"""Cursors on the emulated build (lb_batch_cursor_pos): the engine's answers against the oracle-side reference
(tests/cursor_ref.cpp), field for field, through every import path that takes LB_FLAG_CURSORS; plus the errors, the
refusal on checkouts and the launch counts."""
import os
import random
import subprocess

import pytest

import loro_b200
from loro_b200.api import LB_CURSOR_ID_NOT_FOUND, LB_FLAG_CURSORS, EngineError
from oracle import CT_MOVABLE, OracleDoc

from . import workloads
from .checkout_checks import oracle_doc
from .cursor_checks import cursor_pos_ref, sample_cursors, seq_containers

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")
F = LB_FLAG_CURSORS
EXTRA = ["cid:root-absent:Text", "cid:root-absent:List", "cid:7@1:List"]   # an empty root, a missing normal container


@pytest.fixture(scope="module", autouse=True)
def _emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def check(batch, docs, rnd, k=120):
    """every document i of `batch` (its OracleDoc docs[i]) answers k sampled cursors like the reference, in one call"""
    reqs, want = [], []
    for i, doc in enumerate(docs):
        cs = sample_cursors(rnd, list(seq_containers(doc)) + EXTRA, doc.oplog_vv(), k)
        reqs += [(i,) + c for c in cs]
        want += cursor_pos_ref(doc, cs)
    got = batch.cursor_pos(reqs)
    for r, g, w in zip(reqs, got, want):
        assert g == w, r
    return got


@pytest.mark.parametrize("seed", range(3))
def test_random_histories_fresh_import(seed):
    rnd = random.Random(seed)
    blobs = [workloads.make_doc_history(900 * seed + k, n_sites=rnd.randint(1, 4), n_ops=rnd.randint(60, 300))[0]
             for k in range(6)]
    b = loro_b200.import_batch(blobs, flags=F, lib_path=EMU)
    got = check(b, [oracle_doc([x]) for x in blobs], rnd)
    assert any(u is not None for _, _, _, u in got) and any(s == LB_CURSOR_ID_NOT_FOUND for s, _, _, _ in got)


def test_import_batch_groups_and_split_multibatch():
    rnd = random.Random(5)
    groups = []
    for k in range(4):
        e1, e2, _ = workloads.overlapping_update_blobs(k)
        groups.append([e2, e1] if k % 2 else [e1, e2])
    blobs, ids = [], []
    for i, g in enumerate(groups):
        blobs += g
        ids += [i] * len(g)
    b = loro_b200.import_batch(blobs, doc_ids=ids, flags=F, lib_path=EMU)
    check(b, [oracle_doc(g) for g in groups], rnd)
    single = [workloads.make_doc_history(40 + k, n_sites=3, n_ops=80)[0] for k in range(6)]
    m = loro_b200.import_batch(single, flags=F, lib_path=EMU, split=3)
    assert isinstance(m, loro_b200.api.MultiBatch)
    docs = [oracle_doc([x]) for x in single]
    # requests of every part, interleaved: the answers come back in request order
    reqs = [(i, c) for c in range(3) for i in (5, 0, 3, 1, 4, 2)]
    cs = {i: sample_cursors(rnd, seq_containers(docs[i]), docs[i].oplog_vv(), 3) for i in range(6)}
    got = m.cursor_pos([(i,) + cs[i][c] for i, c in reqs])
    assert got == [cursor_pos_ref(docs[i], [cs[i][c]])[0] for i, c in reqs]


def test_docset_import_rounds_and_read():
    from .docset_checks import _session
    rnd = random.Random(6)
    blobs = _session(4, n_sites=3, rounds=5, edits=12)
    ds = loro_b200.DocSet(lib_path=EMU)
    ref = OracleDoc(9)
    for blob in blobs:
        r = ds.import_([blob], [7], flags=F)
        ref.import_(blob)
        check(r, [ref], rnd, k=60)
    r = ds.read([7, 8], flags=F)
    check(r, [ref, OracleDoc(10)], rnd, k=60)


def test_concurrent_inserts_at_one_position_and_range_deletes():
    """three peers insert at the same place concurrently, then delete ranges forward and backward (a reversed delete
    span), across the concurrent runs"""
    a, b, c = OracleDoc(11), OracleDoc(12), OracleDoc(13)
    ta = a.get_text("t")
    a.text_insert(ta, 0, "base text")
    a.commit()
    for d in (b, c):
        workloads.merge(d, a)
    for d, s in ((a, "AAAA"), (b, "BBBB"), (c, "CCCC")):
        d.text_insert(d.get_text("t"), 4, s)
        la = d.get_list("l")
        d.list_insert(la, 0, *range(5))
        d.commit()
    for x in (a, b, c):
        for y in (a, b, c):
            if x is not y:
                workloads.merge(x, y)
    a.delete(ta, 2, 9)
    a.commit()
    for k in range(6):                       # backspace: one deletion after another, right to left
        a.delete(ta, 8 - k, 1)
    a.commit()
    a.delete(a.get_list("l"), 3, 6)
    a.commit()
    blob = a.export_updates()
    doc = oracle_doc([blob])
    bt = loro_b200.import_batch([blob], flags=F, lib_path=EMU)
    cs = [(cid, (p, ctr), side) for cid in seq_containers(doc) for p in (11, 12, 13) for ctr in range(0, 40)
          for side in (-1, 0, 1)]
    cs += [(cid, None, side) for cid in seq_containers(doc) for side in (-1, 0, 1)]
    assert bt.cursor_pos([(0,) + c for c in cs]) == cursor_pos_ref(doc, cs)


def test_unicode_text():
    a, b = OracleDoc(21), OracleDoc(22)
    t = a.get_text("text")
    a.text_insert(t, 0, "héllo wörld 日本語 🦜🦜 ")
    a.commit()
    workloads.merge(b, a)
    tb = b.get_text("text")
    rnd = random.Random(3)
    for k in range(60):
        d = rnd.choice((a, b))
        tt = t if d is a else tb
        n = d.seq_len(tt)
        d.text_insert(tt, rnd.randint(0, n), rnd.choice(("x", "é", "語", "🦜")))
        if k % 3 == 0 and n > 2:
            d.delete(tt, rnd.randint(0, n - 2), 2)
        d.commit()
        if k % 10 == 0:
            workloads.merge(a, b)
            workloads.merge(b, a)
    workloads.merge(a, b)
    blob = a.export_updates()
    check(loro_b200.import_batch([blob], flags=F, lib_path=EMU), [oracle_doc([blob])], rnd, k=400)


def test_statuses_of_failed_unsupported_and_non_sequence_containers():
    m = OracleDoc(4)
    m.text_insert(m.get_text("text"), 0, "abc")
    m.list_insert(m.container("mlist", CT_MOVABLE), 0, 1)
    m.commit()
    good = OracleDoc(5)
    good.text_insert(good.get_text("text"), 0, "abc")
    good.map_set(good.get_map("m"), "k", 1)
    good.commit()
    ok = good.export_updates()
    bad = ok[:30] + bytes([ok[30] ^ 1]) + ok[31:]
    b = loro_b200.import_batch([m.export_updates(), bad, ok], flags=F, lib_path=EMU)
    assert b.status(0).code == 5 and b.status(1).code != 0
    got = b.cursor_pos([(0, "cid:root-text:Text", None, 0), (1, "cid:root-text:Text", None, 0),
                        (2, "cid:root-m:Map", None, 0), (2, "cid:root-t:Tree", (5, 0), 0),
                        (2, "cid:root-mlist:MovableList", None, 1), (2, "cid:root-text:Text", (5, 1), 1),
                        (2, "cid:root-text:Text", (5, 3), 0)])
    assert [g[0] for g in got] == [6, 1, 1, 1, 1, 0, LB_CURSOR_ID_NOT_FOUND]   # the map op 5@3 is not a text element
    assert got[5] == (0, 1, 1, None)


def test_whole_call_failures_and_empty_call():
    blob = workloads.make_doc_history(2, n_sites=2, n_ops=40)[0]
    plain = loro_b200.import_batch([blob], lib_path=EMU)
    with pytest.raises(EngineError) as e:
        plain.cursor_pos([(0, "cid:root-text:Text", None, 0)])
    assert e.value.status == 1 and "LB_FLAG_CURSORS" in str(e.value)
    b = loro_b200.import_batch([blob], flags=F, lib_path=EMU)
    assert b.cursor_pos([]) == []
    with pytest.raises(EngineError) as e:
        b.cursor_pos([(0, "cid:root-text:Text", None, 0), (1, "cid:root-text:Text", None, 0)])
    assert e.value.status == 1 and "out of range" in str(e.value)
    import ctypes
    from loro_b200 import api
    L = api.load_library(EMU)
    assert L.lb_batch_cursor_pos(b._h, None, 1, (api._CursorResult * 1)()) == 1
    assert L.lb_batch_cursor_pos(b._h, (api._Cursor * 1)(), 1, None) == 1
    c = (api._Cursor * 1)()
    c[0].is_root, c[0].name, c[0].name_len, c[0].type = 1, None, 4, 2
    assert L.lb_batch_cursor_pos(b._h, c, 1, (api._CursorResult * 1)()) == 1
    assert L.lb_batch_cursor_pos(b._h, None, 0, None) == 0
    assert b.timings()["cursors"] >= 0
    del ctypes


def test_checkout_entry_points_refuse_the_flag():
    blob = workloads.make_doc_history(3, n_sites=2, n_ops=40)[0]
    with pytest.raises(EngineError) as e:
        loro_b200.import_batch_at([blob], {0: []}, flags=F, lib_path=EMU)
    assert e.value.status == 1
    ds = loro_b200.DocSet(lib_path=EMU)
    ds.import_([blob], [1])
    with pytest.raises(EngineError) as e:
        ds.checkout([(1, [])], flags=F)
    assert e.value.status == 1


def _traced_kernels(capfd):
    return [line.split()[2] for line in capfd.readouterr().err.splitlines() if line.startswith("simt_emu: launch ")]


def test_launch_counts(monkeypatch, capfd):
    """without the flag nothing more is launched; with it one launch at import, and one per query call whatever the
    number of cursors and documents"""
    monkeypatch.setenv("LB_EMU_KTRACE", "1")
    for n in (1, 5):
        blobs = [workloads.make_doc_history(700 + k, n_sites=2, n_ops=50)[0] for k in range(n)]
        capfd.readouterr()
        plain = loro_b200.import_batch(blobs, lib_path=EMU)
        k0 = _traced_kernels(capfd)
        cur = loro_b200.import_batch(blobs, flags=F, lib_path=EMU)
        k1 = _traced_kernels(capfd)
        assert not any("k_cursor" in k for k in k0)
        assert plain.timings()["kernel_launches"] == len(k0)
        assert cur.timings()["kernel_launches"] == len(k1) == len(k0) + 1
        assert sum("k_cursor_tables" in k for k in k1) == 1
        for m in (1, 37 * n):
            cur.cursor_pos([(i % n, "cid:root-text:Text", None, 1) for i in range(m)])
            k2 = _traced_kernels(capfd)
            assert len(k2) == 1 and "k_cursor_query" in k2[0]
        assert cur.timings()["kernel_launches"] == len(k1) + 2
