"""The cursor reference (tests/cursor_ref.cpp) pinned to the reference's own answers (crates/loro/tests/loro_rust_test.rs
get_cursor, get_cursor_at_the_end, get_cursor_for_list; updates stand in for the snapshot, the rich-text mark step is
left out), and checked on random histories against independent sources: the attribution reference's runs
(tests/attribution_checks.py) and the deep value."""
import random

import pytest

from oracle import OracleDoc

from . import workloads
from .checkout_checks import oracle_doc
from .cursor_checks import cursor_pos_ref, sample_cursors, seq_containers

TEXT = "cid:root-text:Text"
LIST = "cid:root-list:List"


def pos_of(doc, cursor):
    status, pos, side, update = cursor_pos_ref(doc, [cursor])[0]
    assert status == 0
    return pos, side, update


def test_get_cursor():
    d1 = OracleDoc(1)
    t1 = d1.get_text("text")
    d1.text_insert(t1, 0, "6789")
    d1.commit()
    pos_7 = (TEXT, (1, 1), 0)          # text.get_cursor(1): the id of '7', Side::Middle
    assert pos_of(d1, pos_7) == (1, 0, None)
    d1.text_insert(t1, 0, "012345")
    d1.commit()
    assert pos_of(d1, pos_7) == (7, 0, None)
    d2 = OracleDoc(2)
    t2 = d2.get_text("text")
    d2.text_insert(t2, 0, "ab")
    d2.commit()
    pos_a = (TEXT, (2, 0), 0)
    assert pos_of(d2, pos_a) == (0, 0, None)
    d2.import_(d1.export_updates())
    assert d2.get_deep_value() == {"text": "0123456789ab"}
    assert pos_of(d2, pos_a) == (10, 0, None)
    d2.delete(t2, 5, 5)
    d2.commit()
    # '7' is deleted: the visible elements before it, Side::Left, and the update cursor at 'a' (2@0)
    assert pos_of(d2, pos_7) == (5, -1, ((2, 0), -1, 5))


def test_get_cursor_at_the_end():
    d = OracleDoc(5)
    t = d.get_text("text")
    d.text_insert(t, 0, "01234")
    d.commit()
    at_end = (TEXT, None, 1)           # text.get_cursor(5) at the end: no id, Side::Right
    want = []
    for step in range(4):
        if step == 1:
            d.text_insert(t, 0, "01234")
        elif step == 2:
            d.delete(t, 0, 10)
        elif step == 3:
            d.text_insert(t, 0, "01234")
        d.commit()
        want.append(pos_of(d, at_end)[0])
    assert want == [5, 10, 0, 5]


def test_get_cursor_for_list():
    d = OracleDoc(7)
    lst = d.get_list("list")
    pos_start = (LIST, None, -1)       # list.get_cursor(0) on the empty list: no id, Middle becomes Left
    d.list_insert(lst, 0, 1)
    d.commit()
    pos_0 = (LIST, (7, 0), 0)
    pos_end = (LIST, None, 1)
    for k in range(4):
        assert [pos_of(d, c)[0] for c in (pos_start, pos_0, pos_end)] == [0, k, k + 1]
        d.list_insert(lst, 0, 1)
        d.commit()


def test_empty_and_missing_containers():
    d = OracleDoc(3)
    d.text_insert(d.get_text("text"), 0, "abc")
    d.commit()
    # a root container no op touches is empty; a normal container the document lacks does not exist
    assert cursor_pos_ref(d, [("cid:root-none:Text", None, 1), ("cid:root-none:List", (3, 0), 0),
                              ("cid:0@3:Text", None, -1), ("cid:root-text:Map", None, 0)]) == [
        (0, 0, 1, None), (100, 0, 0, None), (100, 0, -1, None), (1, 0, 0, None)]


@pytest.mark.parametrize("seed", range(6))
def test_invariants_on_random_three_peer_histories(seed):
    rnd = random.Random(seed)
    blob = workloads.make_doc_history(300 + seed, n_sites=3, n_ops=rnd.randint(150, 400))[0]
    doc = oracle_doc([blob])
    runs = seq_containers(doc)
    deep = doc.get_deep_value()
    for cid, ids in runs.items():
        name = cid[len("cid:root-"):].rsplit(":", 1)[0]
        if cid.startswith("cid:root-") and name in deep:
            assert len(ids) == len(deep[name])
    cursors = sample_cursors(rnd, runs, doc.oplog_vv(), 600)
    n_deleted = 0
    for (cid, tid, side), (status, pos, rside, update) in zip(cursors, cursor_pos_ref(doc, cursors)):
        ids = runs[cid]
        assert pos <= len(ids)
        if tid is None:
            assert (status, pos, rside, update) == (0, 0 if side == -1 else len(ids), side, None)
        elif tid in ids:
            assert (status, pos, rside, update) == (0, ids.index(tid), side, None)
        elif status == 0:
            n_deleted += 1
            assert rside == -1
            assert update == ((ids[pos], -1, pos) if pos < len(ids) else (None, 1, len(ids)) if ids else (None, -1, 0))
        else:
            assert status == 100
    assert n_deleted > 0
