"""Checkout on the emulated build: the state of documents at requested frontiers (lb_import_batch_at, lb_docset_checkout)
against the oracle's capped replay, JSON byte for byte."""
import ctypes
import json
import os
import random
import subprocess

import pytest

import loro_b200
from loro_b200.api import EngineError
from oracle import OracleDoc

from . import workloads
from .checkout_checks import (FRONTIERS_NOT_FOUND, applied_ids, check_import_batch_at, interesting_ids, json_at,
                              oracle_doc, random_frontiers)

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def test_version_layout_matches_the_c_compiler(tmp_path):
    """the ctypes mirror of lb_version against the C compiler's layout of include/loro_b200.h"""
    from loro_b200.api import _Version
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "loro_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(lb_version), offsetof(lb_version, doc_id),\n'
                   '         offsetof(lb_version, frontiers), offsetof(lb_version, n_frontiers));\n'
                   '  printf("%d\\n", (int)LB_DOC_ERR_FRONTIERS);\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(os.path.dirname(HERE), "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split()
    assert [int(x) for x in out[:4]] == [ctypes.sizeof(_Version), _Version.doc_id.offset, _Version.frontiers.offset,
                                         _Version.n_frontiers.offset]
    assert int(out[4]) == FRONTIERS_NOT_FOUND == 7
    assert loro_b200.api.DOC_CODES[7] == "FrontiersNotFound"


@pytest.mark.parametrize("seed", range(4))
def test_random_histories_at_random_ids(seed):
    """mixed Text / List / Map histories (child containers, nested values), each document at a random applied id or a
    multi-id frontier with redundant ids, ids inside changes and inside inserts and delete spans included"""
    rnd = random.Random(seed)
    groups, requests = [], {}
    for k in range(10):
        blob, _, _, _ = workloads.make_doc_history(1000 * seed + k, n_sites=rnd.randint(1, 4), n_ops=rnd.randint(40, 160))
        groups.append([blob])
        o = oracle_doc([blob])
        inside = interesting_ids(blob)
        if k % 3 == 0 and inside:
            requests[k] = [rnd.choice(inside)]
        elif k % 3 == 1:
            requests[k] = random_frontiers(rnd, o, max_ids=4)
        elif k != 8:
            requests[k] = [rnd.choice(applied_ids(o))]
    check_import_batch_at(groups, requests, lib_path=EMU)


def test_every_id_inside_ops_of_one_document():
    """one document at each of its ids that cut a change or an op (text / list inserts, forward and reversed deletes)"""
    blob, _, _, _ = workloads.make_doc_history(77, n_sites=2, n_ops=120)
    ids = interesting_ids(blob)
    assert len(ids) > 10
    o = oracle_doc([blob])
    ds = loro_b200.DocSet(lib_path=EMU)
    ds.import_([blob], [5])
    r = ds.checkout([(5, [i]) for i in ids])
    for k, i in enumerate(ids):
        assert r.status(k).code == 0, i
        assert r.json_bytes(k) == json_at(o, [i]), i


def test_reversed_and_forward_delete_spans_cut_at_the_tail():
    """deletes typed backwards (a reversed DeleteSpanWithId) and forwards, checked out at every id inside them: the tail
    cut moves the start of a reversed span only (list_op.rs:251-270), and atoms never integrated are never toggled"""
    a, b = OracleDoc(1), OracleDoc(2)
    t = a.get_text("text")
    a.text_insert(t, 0, "0123456789abcdefghij")
    a.commit()
    workloads.merge(b, a)
    for k in range(6):                         # backspace x6: one reversed span
        a.delete(t, 15 - k, 1)
    a.commit()
    tb = b.get_text("text")
    for _ in range(5):                         # forward delete x5 at one position: one forward span
        b.delete(tb, 2, 1)
    b.text_insert(tb, 2, "XY")
    b.commit()
    workloads.merge(a, b)
    blob = a.export_updates()
    o = oracle_doc([blob])
    ids = applied_ids(o)
    ds = loro_b200.DocSet(lib_path=EMU)
    ds.import_([blob], [1])
    reqs = [(1, [i]) for i in ids] + [(1, [(1, 23), (2, 3)]), (1, [(1, 22), (2, 6)]), (1, [(2, 1), (1, 18)])]
    r = ds.checkout(reqs)
    for k, (_, f) in enumerate(reqs):
        assert r.status(k).code == 0, f
        assert r.json_bytes(k) == json_at(o, f), f


def test_empty_and_oplog_frontiers():
    blobs = [workloads.make_doc_history(300 + k, n_sites=3, n_ops=100)[0] for k in range(3)]
    plain = loro_b200.import_batch(blobs, lib_path=EMU)
    fr = {k: plain.oplog_frontiers(k) for k in range(3)}
    r = loro_b200.import_batch_at(blobs, {0: [], 1: fr[1]}, lib_path=EMU)
    assert r.status(0).code == 0 and r.json_bytes(0) == json_at(oracle_doc([blobs[0]]), [])
    assert r.json_bytes(1) == plain.json_bytes(1)          # the oplog frontiers: the latest state, byte for byte
    assert r.json_bytes(2) == plain.json_bytes(2)          # not named: the latest state
    assert r.oplog_vv(0) == plain.oplog_vv(0) and r.oplog_frontiers(0) == fr[0]
    assert r.status(0).success == plain.status(0).success


@pytest.mark.parametrize("seed", range(2))
def test_tree_histories(seed):
    """C5-shaped movable-tree histories (concurrent moves, cycles, deletes, meta maps) at random ids"""
    rnd = random.Random(seed)
    groups, requests = [], {}
    for k in range(6):
        blob, _, _, _ = workloads.make_tree_history(50 * seed + k, n_sites=3, n_base=20, n_ops=60, mixed=k % 2 == 1)
        groups.append([blob])
        requests[k] = random_frontiers(rnd, oracle_doc([blob]), max_ids=2)
    check_import_batch_at(groups, requests, lib_path=EMU)


def test_import_batch_groups_with_overlapping_blobs():
    """documents of several blobs whose changes overlap partially (trimmed copies): the id is found in whichever copy
    applied it"""
    rnd = random.Random(5)
    groups, requests = [], {}
    for k in range(4):
        e1, e2, n = workloads.overlapping_update_blobs(k)
        assert n > 0
        groups.append([e2, e1] if k % 2 else [e1, e2])
        o = oracle_doc(groups[-1])
        requests[k] = [rnd.choice(interesting_ids(e2) + applied_ids(o))]
    check_import_batch_at(groups, requests, lib_path=EMU)


def test_unsupported_ops_are_decided_over_the_whole_history():
    """a document with a movable-list op (unsupported) in the middle of its history: code 5 wherever the checkout cuts --
    before the op, at it, after it, at the empty version -- exactly as lb_import_batch reports it"""
    from oracle import CT_MOVABLE
    d = OracleDoc(3)
    d.text_insert(d.get_text("text"), 0, "hello")
    d.commit()
    blob_ok = d.export_updates()
    m = OracleDoc(4)
    mt = m.get_text("text")
    m.text_insert(mt, 0, "abc")
    m.commit()
    m.list_insert(m.container("mlist", CT_MOVABLE), 0, 1)
    m.commit()
    m.text_insert(mt, 3, "def")
    m.commit()
    blob_un = m.export_updates()
    plain = loro_b200.import_batch([blob_un, blob_ok], lib_path=EMU)
    assert plain.status(0).code == 5 and plain.status(1).code == 0
    for f in ([(4, 0)], [(4, 2)], [(4, 3)], [], [(4, 6)]):
        r = loro_b200.import_batch_at([blob_un, blob_ok], {0: f}, lib_path=EMU)
        assert r.status(0).code == 5, f
        assert r.status(1).code == 0 and r.json_bytes(1) == plain.json_bytes(1)


def test_ids_outside_the_dag_fail_that_document_only():
    """an unknown peer, a counter at or past the vv, a pending change's id: code 7 (FrontiersNotFound); the other
    documents of the batch are unaffected"""
    a = OracleDoc(1)
    t = a.get_text("text")
    a.text_insert(t, 0, "abc")
    a.commit()
    u1 = a.export_updates()
    a.text_insert(t, 3, "def")
    a.commit()
    u2 = a.export_updates({1: 3})
    blobs = [workloads.make_doc_history(k, n_sites=2, n_ops=60)[0] for k in range(2)]
    groups = [[blobs[0]], [u2], [u1], [blobs[1]], [u2, u1]]
    vv0 = oracle_doc([blobs[0]]).oplog_vv()
    peer0 = next(iter(vv0))
    requests = {0: [(peer0, vv0[peer0])],      # counter at the vv
                1: [(1, 4)],                   # inside a pending change
                2: [(424242, 0)],              # unknown peer
                4: [(1, 4), (1, 1)]}           # the same change released by the second blob: found
    batch = check_import_batch_at(groups, requests, lib_path=EMU,
                                  expect_codes={0: FRONTIERS_NOT_FOUND, 1: FRONTIERS_NOT_FOUND, 2: FRONTIERS_NOT_FOUND, 4: 0})
    assert batch.status(3).code == 0
    assert batch.json_bytes(4) == b'{"text":"abcde"}'
    assert batch.oplog_vv(0) == vv0


def test_argument_errors():
    blob = workloads.make_doc_history(1, n_sites=2, n_ops=20)[0]
    L = loro_b200.load_library(EMU)
    from loro_b200.api import LB_FLAG_COMPACT, LB_FLAG_EXPORT, _Options, _Version, _blob_array, _version_array
    for versions, flags in (({7: []}, 0),                        # a doc_id no blob carries
                            ({0: []}, LB_FLAG_EXPORT), ({0: []}, LB_FLAG_COMPACT)):
        with pytest.raises(EngineError) as e:
            loro_b200.import_batch_at([blob], versions, flags=flags, lib_path=EMU)
        assert e.value.status == 1
    arr, keep = _blob_array([blob], None)
    ver, vkeep = _version_array([(0, [(1, 0)]), (0, [])])          # named twice
    h = ctypes.c_void_p()
    opt = _Options(device=0, flags=0)
    assert L.lb_import_batch_at(arr, 1, ver, 2, ctypes.byref(opt), ctypes.byref(h)) == 1
    nul = (_Version * 1)()
    nul[0].doc_id = 0
    nul[0].n_frontiers = 2                                        # null frontiers with n > 0
    assert L.lb_import_batch_at(arr, 1, nul, 1, ctypes.byref(opt), ctypes.byref(h)) == 1
    ds = loro_b200.DocSet(lib_path=EMU)
    ds.import_([blob], [0])
    assert L.lb_docset_checkout(ds._h, nul, 1, ctypes.byref(opt), ctypes.byref(h)) == 1
    with pytest.raises(EngineError):
        ds.checkout([(0, [])], flags=LB_FLAG_EXPORT)
    r = loro_b200.import_batch_at([blob], {0: []}, lib_path=EMU)
    with pytest.raises(EngineError) as e:
        r.export_updates(0)
    assert e.value.status == 1


def test_docset_history_browsing():
    """after each import of a stream, record (oplog frontiers, json); later every recorded version checks out to that JSON,
    and the set's stored bytes, document count and later exports are unchanged by the checkouts"""
    from .docset_checks import _session
    blobs = _session(3, n_sites=3, rounds=6, edits=10)
    ds = loro_b200.DocSet(lib_path=EMU)
    ref = OracleDoc(9)
    seen = []
    for k, blob in enumerate(blobs):
        r = ds.import_([blob], [11])
        ref.import_(blob)
        assert r.json_bytes(0) == ref.json_text()
        if ref.pending_count() == 0:
            seen.append((r.oplog_frontiers(0), r.json_bytes(0)))
    assert len(seen) > 4
    stored, n = ds.stored_bytes, ds.n_docs
    reqs = [(11, f) for f, _ in seen] + [(99, [])]
    r = ds.checkout(reqs)
    assert r.n_docs == len(reqs)
    for k, (f, js) in enumerate(seen):
        st = r.status(k)
        assert st.code == 0 and st.success == {} and st.pending is None, (k, st)
        got = r.json_bytes(k)
        assert got == json_at(ref, f), (k, f)
        # the recording, except for root containers the document registered later: they are listed, empty
        # (state.rs:894-924 iterates every registered root)
        later = {key: v for key, v in json.loads(got).items() if key not in json.loads(js)}
        assert all(v in ("", [], {}) for v in later.values()), later
        assert {key: v for key, v in json.loads(got).items() if key not in later} == json.loads(js), (k, f)
        assert r.oplog_vv(k) == ref.oplog_vv()
    assert r.status(len(seen)).code == 0 and r.json_bytes(len(seen)) == b"{}"   # a doc_id the set has never seen
    assert ds.stored_bytes == stored and ds.n_docs == n
    last = workloads.make_doc_history(5, n_sites=2, n_ops=20)[0]
    r2 = ds.import_([last], [11])
    ref.import_(last)
    assert r2.json_bytes(0) == ref.json_text() and r2.export_updates(0) == ref.export_updates()
