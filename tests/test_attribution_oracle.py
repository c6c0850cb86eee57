"""The attribution reference (tests/attribution_ref.cpp) pinned against the reference's own known answers
(crates/loro/tests/loro_rust_test.rs get_last_editor_on_map, get_editor) and against the deep value on random histories."""
import json
import random

import pytest

from oracle import OracleDoc

from . import workloads
from .attribution_checks import attribution_at, parsed


def _containers(doc):
    peers, cs = parsed(attribution_at(doc))
    return peers, cs


def _editor_at(peers, runs, pos):
    """the peer that inserted the element at `pos` (get_editor_at_unicode_pos / get_id_at(pos).peer)"""
    for p, c, n in runs:
        if pos < n:
            return peers[p], c + pos
        pos -= n
    return None


def test_get_last_editor_on_map():
    """loro_rust_test.rs:2262: key1 is written by peer 0, then by peer 1; key2 by peer 1; a missing key has no entry"""
    d = OracleDoc(0)
    m = d.get_map("map")
    d.map_set(m, "key1", "value1")
    d.commit()
    peers, cs = _containers(d)
    assert peers[cs["cid:root-map:Map"]["key1"][0]] == 0
    d.set_peer_id(1)
    d.map_set(m, "key1", "value2")
    d.map_set(m, "key2", "value3")
    d.commit()
    peers, cs = _containers(d)
    entry = cs["cid:root-map:Map"]
    assert peers[entry["key1"][0]] == 1 and peers[entry["key2"][0]] == 1
    assert "nonexistent" not in entry
    assert entry["key1"][2] == 1 and entry["key2"][2] == 1


def test_get_editor_text_list_and_tree_moves():
    """loro_rust_test.rs:2279 without its movable-list part: text position 3 and list position 0 are peer 0's; the tree
    node's last move is peer 1's creation, then peer 2's move"""
    d = OracleDoc(0)
    t = d.get_text("text")
    d.text_insert(t, 0, "01234")
    lst = d.get_list("list")
    d.list_insert(lst, 0, 0)
    d.commit()
    peers, cs = _containers(d)
    assert _editor_at(peers, cs["cid:root-text:Text"], 3) == (0, 3)
    assert _editor_at(peers, cs["cid:root-list:List"], 0)[0] == 0
    d.set_peer_id(1)
    tree = d.get_tree("tree")
    n0 = d.tree_create(tree)
    n1 = d.tree_create(tree)
    d.commit()
    peers, cs = _containers(d)
    key = "%d@%d" % (n0[1], n0[0])
    p, ctr, alive = cs["cid:root-tree:Tree"][key]
    assert peers[p] == 1 and (peers[p], ctr) == n0 and alive == 1     # the creation is the last move
    d.set_peer_id(2)
    d.tree_move(tree, n0, parent=n1)
    d.commit()
    peers, cs = _containers(d)
    p, ctr, alive = cs["cid:root-tree:Tree"][key]
    assert peers[p] == 2 and ctr == 0 and alive == 1
    assert peers[cs["cid:root-tree:Tree"]["%d@%d" % (n1[1], n1[0])][0]] == 1


def test_deleted_keys_and_nodes_keep_their_editor():
    d = OracleDoc(5)
    m = d.get_map("m")
    d.map_set(m, "a", 1)
    d.map_set(m, "b", 2)
    d.commit()
    tree = d.get_tree("t")
    n = d.tree_create(tree)
    d.commit()
    d.set_peer_id(6)
    d.map_delete(m, "a")
    d.tree_delete(tree, n)
    d.commit()
    peers, cs = _containers(d)
    assert peers == [5, 6]
    a = cs["cid:root-m:Map"]["a"]
    assert peers[a[0]] == 6 and a[2] == 0 and cs["cid:root-m:Map"]["b"][2] == 1
    p, ctr, alive = cs["cid:root-t:Tree"]["%d@%d" % (n[1], n[0])]
    assert peers[p] == 6 and alive == 0


def _tree_ids(nodes):
    out = set()
    for n in nodes:
        out.add(n["id"])
        out |= _tree_ids(n["children"])
    return out


@pytest.mark.parametrize("seed", range(6))
def test_invariants_on_random_histories(seed):
    """run lengths sum to the text / list length of the deep value, the present keys of a root map are exactly its deep
    value's keys, the alive nodes of a root tree exactly its deep value's nodes, and every id is a distinct atom"""
    rnd = random.Random(seed)
    if seed % 2:
        blob = workloads.make_tree_history(seed, n_sites=3, n_base=20, n_ops=80, mixed=True)[0]
    else:
        blob = workloads.make_doc_history(seed, n_sites=rnd.randint(1, 5), n_ops=200)[0]
    d = OracleDoc(1)
    d.import_(blob)
    deep = json.loads(d.json_text())
    peers, cs = _containers(d)
    assert peers == sorted(d.oplog_vv())
    for name, value in deep.items():
        if isinstance(value, str):
            runs = cs.get("cid:root-%s:Text" % name, [])
            assert sum(n for _, _, n in runs) == len(value)
        elif isinstance(value, dict):
            entry = cs.get("cid:root-%s:Map" % name, {})
            assert {k for k, (_, _, f) in entry.items() if f} == set(value)
        elif "cid:root-%s:Tree" % name in cs:
            entry = cs["cid:root-%s:Tree" % name]
            assert {k for k, (_, _, f) in entry.items() if f} == _tree_ids(value)
        else:
            runs = cs.get("cid:root-%s:List" % name, [])
            assert sum(n for _, _, n in runs) == len(value)
    for cid, entry in cs.items():
        if isinstance(entry, list):
            ids = [(peers[p], c + k) for p, c, n in entry for k in range(n)]
            assert len(ids) == len(set(ids)), cid
            for a, b in zip(entry, entry[1:]):     # maximal runs
                assert not (a[0] == b[0] and a[1] + a[2] == b[1]), cid
