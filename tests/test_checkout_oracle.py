"""The checkout reference (tests/checkout_ref.cpp: the oracle's replay capped at the causal closure of F) against known
answers of the reference and against a second formulation: what a site itself showed at the moment its frontiers were F."""
import json

import pytest

from oracle import OracleDoc

from . import workloads
from .checkout_checks import history_snapshots, json_at


def test_typed_insert_cut_inside_the_op():
    """"Hello" typed as one insert by peer 1, checked out at [(1, 2)], reads "Hel": the op under the cut is cut inside"""
    d = OracleDoc(1)
    d.text_insert(d.get_text("text"), 0, "Hello")
    d.commit()
    assert json_at(d, [(1, 2)]) == b'{"text":"Hel"}'
    assert json_at(d, [(1, 4)]) == d.json_text()
    assert json_at(d, []) == b'{"text":""}'


def test_list_checkout_known_answers():
    """loro_rust_test.rs:129-170 list_checkout: a list of a text container and a map container; the states at the
    frontiers after each step, every root container listed whether or not it has ops inside F"""
    d = OracleDoc(0)
    lst = d.get_list("list")
    d.list_insert_container(lst, 0, 0)        # map at 0
    d.commit()
    f0 = d.frontiers()
    d.list_insert_container(lst, 0, 2)        # text at 0
    d.commit()
    f1 = d.frontiers()
    d.delete(lst, 1, 1)
    d.commit()
    f2 = d.frontiers()
    d.delete(lst, 0, 1)
    d.commit()
    assert json.loads(json_at(d, f1)) == {"list": ["", {}]}
    assert json.loads(json_at(d, f2)) == {"list": [""]}
    assert json.loads(json_at(d, f0)) == {"list": [{}]}
    assert json.loads(json_at(d, [])) == {"list": []}


def test_checkout_to_unknown_version():
    """loro_rust_test.rs:3542 test_checkout_to_unknown_version: ids outside the DAG are FrontiersNotFound -- an unknown
    peer, a counter at or past the vv, an id of a change that is still pending"""
    a, b = OracleDoc(1), OracleDoc(2)
    a.text_insert(a.get_text("text"), 0, "abc")
    a.commit()
    u1 = a.export_updates()
    a.text_insert(a.get_text("text"), 3, "def")
    a.commit()
    u2 = a.export_updates({1: 3})
    b.import_(u2)                              # pending: its dependency (1, 2) is missing
    assert b.pending_count() > 0
    assert json_at(b, [(1, 4)]) is None
    assert json_at(b, [(7, 0)]) is None
    b.import_(u1)
    assert json_at(b, [(1, 4)]) == b'{"text":"abcde"}'
    assert json_at(b, [(1, 6)]) is None
    assert json_at(b, [(1, -1)]) is None


def test_redundant_ids_are_shrunk():
    """shrink_frontiers: an id in the causal past of another changes nothing"""
    d = OracleDoc(1)
    t = d.get_text("text")
    d.text_insert(t, 0, "abcdef")
    d.commit()
    assert json_at(d, [(1, 1), (1, 4), (1, 0)]) == json_at(d, [(1, 4)]) == b'{"text":"abcde"}'


@pytest.mark.parametrize("seed", range(6))
def test_capped_replay_equals_what_the_site_showed(seed):
    blob, snaps = history_snapshots(seed, n_sites=3, n_ops=160)
    assert len(snaps) > 5
    full = OracleDoc(1)
    full.import_(blob)
    site_view = OracleDoc(2)                   # registers the same root containers as every site did
    site_view.get_text("text"), site_view.get_list("list"), site_view.get_map("map")
    site_view.import_(blob)
    for frontiers, js in snaps:
        assert json_at(site_view, frontiers) == js, frontiers
    assert json_at(full, full.frontiers()) == full.json_text()


@pytest.mark.parametrize("seed", range(3))
def test_capped_replay_of_trees_equals_what_the_site_showed(seed):
    blob, snaps = history_snapshots(100 + seed, n_sites=3, n_ops=120, tree=True)
    site_view = OracleDoc(2)
    site_view.get_text("text"), site_view.get_list("list"), site_view.get_map("map"), site_view.get_tree("tree")
    site_view.import_(blob)
    for frontiers, js in snaps:
        assert json_at(site_view, frontiers) == js, frontiers


def test_oplog_frontiers_equal_the_latest_state():
    for seed in range(4):
        blob, js, _, _ = workloads.make_doc_history(seed, n_sites=3, n_ops=120)
        d = OracleDoc(1)
        d.import_(blob)
        assert json_at(d, d.frontiers()) == js
