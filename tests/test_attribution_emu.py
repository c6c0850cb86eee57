"""Attribution on the emulated build (lb_doc_attribution): the engine's bytes against the oracle-side reference
(tests/attribution_ref.cpp), byte for byte, through every import path; plus the call's errors and launch count."""
import os
import random
import subprocess

import pytest

import loro_b200
from loro_b200.api import LB_FLAG_ATTRIBUTION, LB_FLAG_EXPORT, LB_FLAG_NO_JSON, EngineError
from oracle import CT_MOVABLE, OracleDoc

from . import workloads
from .attribution_checks import attribution_at
from .checkout_checks import interesting_ids, oracle_doc, random_frontiers

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")
A = LB_FLAG_ATTRIBUTION


@pytest.fixture(scope="module", autouse=True)
def _emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def check_groups(groups, flags=A):
    """document i = import_batch(groups[i]): engine bytes == the reference's at the latest version"""
    blobs, ids = [], []
    for i, g in enumerate(groups):
        blobs += list(g)
        ids += [i] * len(g)
    b = loro_b200.import_batch(blobs, doc_ids=ids, flags=flags, lib_path=EMU)
    for i, g in enumerate(groups):
        assert b.status(i).code == 0, i
        assert b.attribution_bytes(i) == attribution_at(oracle_doc(g)), i
    return b


@pytest.mark.parametrize("seed", range(4))
def test_random_histories_one_to_five_sites(seed):
    rnd = random.Random(seed)
    check_groups([[workloads.make_doc_history(500 * seed + k, n_sites=rnd.randint(1, 5), n_ops=rnd.randint(40, 250))[0]]
                  for k in range(8)])


@pytest.mark.parametrize("seed", range(2))
def test_tree_histories(seed):
    """concurrent moves, cycles, deletes (deleted nodes keep an entry), meta maps"""
    check_groups([[workloads.make_tree_history(70 * seed + k, n_sites=3, n_base=25, n_ops=80, mixed=k % 2 == 1)[0]]
                  for k in range(6)])


def test_multi_byte_text_and_long_runs():
    """unicode scalar values (2-, 3- and 4-byte UTF-8) and a text of many runs, merged across chunks of 32 runs"""
    a, b = OracleDoc(11), OracleDoc(12)
    t = a.get_text("text")
    a.text_insert(t, 0, "héllo wörld 日本語 🦜🦜 " * 3)
    a.commit()
    workloads.merge(b, a)
    tb = b.get_text("text")
    rnd = random.Random(3)
    for k in range(120):
        d = rnd.choice((a, b))
        tt = t if d is a else tb
        n = d.seq_len(tt)
        d.text_insert(tt, rnd.randint(0, n), rnd.choice(("x", "é", "語", "🦜", "ab")))
        if k % 7 == 0 and n > 2:
            d.delete(tt, rnd.randint(0, n - 2), 1)
        d.commit()
        if k % 10 == 0:
            workloads.merge(a, b)
            workloads.merge(b, a)
    workloads.merge(a, b)
    check_groups([[a.export_updates()]])


def test_nested_containers_and_containers_under_deleted_keys():
    """child containers of maps and lists; a child whose map entry was deleted or overwritten keeps its entries"""
    d = OracleDoc(21)
    m = d.get_map("root")
    child = d.map_set_container(m, "child", 2)          # Text
    d.text_insert(child, 0, "inner")
    sub = d.map_set_container(m, "sub", 0)              # Map
    d.map_set(sub, "k", 1)
    lst = d.get_list("l")
    inner = d.list_insert_container(lst, 0, 1)          # List
    d.list_insert(inner, 0, 1, 2, 3)
    d.commit()
    d.set_peer_id(22)
    d.map_delete(m, "child")
    d.map_set(m, "sub", "overwritten")
    d.text_insert(child, 5, "!")
    d.commit()
    b = check_groups([[d.export_updates()]])
    cids = list(b.attribution(0))
    assert cids[:2] == ["cid:root-l:List", "cid:root-root:Map"] and len(cids) == 5


def test_import_batch_groups_with_overlapping_blobs():
    groups = []
    for k in range(4):
        e1, e2, _ = workloads.overlapping_update_blobs(k)
        groups.append([e2, e1] if k % 2 else [e1, e2])
    check_groups(groups)


def test_pending_changes():
    """a blob whose dependencies are missing is parked: its changes attribute nothing, and the peers list is the oplog
    vv's"""
    a = OracleDoc(31)
    t = a.get_text("t")
    a.text_insert(t, 0, "abc")
    a.commit()
    u1 = a.export_updates()
    vv = a.oplog_vv()
    a.set_peer_id(32)
    a.text_insert(t, 3, "def")
    a.commit()
    u2 = a.export_updates(vv)
    b = check_groups([[u2], [u1], [u2, u1]])
    assert b.attribution_bytes(0) == b'{"peers":[],"containers":{}}'


def test_docset_imports_and_read():
    from .docset_checks import _session
    blobs = _session(4, n_sites=3, rounds=5, edits=10)
    ds = loro_b200.DocSet(lib_path=EMU)
    ref = OracleDoc(9)
    for blob in blobs:
        r = ds.import_([blob], [7], flags=A)
        ref.import_(blob)
        assert r.attribution_bytes(0) == attribution_at(ref)
    r = ds.read([7, 8], flags=A)
    assert r.attribution_bytes(0) == attribution_at(ref)
    assert r.attribution_bytes(1) == b'{"peers":[],"containers":{}}'


@pytest.mark.parametrize("seed", range(3))
def test_import_batch_at_and_docset_checkout_at_random_frontiers(seed):
    rnd = random.Random(seed)
    blobs, requests = [], {}
    for k in range(6):
        if k % 3 == 2:
            blob = workloads.make_tree_history(90 * seed + k, n_sites=3, n_base=15, n_ops=50)[0]
        else:
            blob = workloads.make_doc_history(90 * seed + k, n_sites=rnd.randint(1, 4), n_ops=rnd.randint(40, 150))[0]
        blobs.append(blob)
        o = oracle_doc([blob])
        inside = interesting_ids(blob)
        requests[k] = [rnd.choice(inside)] if k % 2 and inside else random_frontiers(rnd, o, max_ids=3)
    b = loro_b200.import_batch_at(blobs, requests, flags=A, lib_path=EMU)
    for k, blob in enumerate(blobs):
        assert b.status(k).code == 0, k
        assert b.attribution_bytes(k) == attribution_at(oracle_doc([blob]), requests[k]), (k, requests[k])
    ds = loro_b200.DocSet(lib_path=EMU)
    ds.import_([blobs[0]], [1])
    o = oracle_doc([blobs[0]])
    fs = [random_frontiers(rnd, o, max_ids=2) for _ in range(5)] + [[]]
    r = ds.checkout([(1, f) for f in fs], flags=A)
    for k, f in enumerate(fs):
        assert r.attribution_bytes(k) == attribution_at(o, f), f


def test_unsupported_and_failed_documents_follow_lb_doc_json():
    m = OracleDoc(4)
    m.text_insert(m.get_text("text"), 0, "abc")
    m.list_insert(m.container("mlist", CT_MOVABLE), 0, 1)
    m.commit()
    good = workloads.make_doc_history(1, n_sites=2, n_ops=40)[0]
    bad = good[:30] + bytes([good[30] ^ 1]) + good[31:]
    b = loro_b200.import_batch([m.export_updates(), bad, good], flags=A, lib_path=EMU)
    assert b.status(0).code == 5 and b.status(1).code != 0
    assert b.attribution_bytes(0) == b.json_bytes(0) == b""
    assert b.attribution_bytes(1) == b.json_bytes(1) == b""
    assert b.attribution_bytes(2) == attribution_at(oracle_doc([good]))


def test_flag_required_and_independent_of_no_json_and_export():
    blob = workloads.make_doc_history(2, n_sites=3, n_ops=80)[0]
    want = attribution_at(oracle_doc([blob]))
    b = loro_b200.import_batch([blob], lib_path=EMU)
    with pytest.raises(EngineError) as e:
        b.attribution_bytes(0)
    assert e.value.status == 1 and "LB_FLAG_ATTRIBUTION" in str(e.value)
    with pytest.raises(EngineError):
        b.attribution_bytes(1)
    b = loro_b200.import_batch([blob], flags=A | LB_FLAG_NO_JSON, lib_path=EMU)
    assert b.attribution_bytes(0) == want
    with pytest.raises(EngineError):
        b.json_bytes(0)
    b = loro_b200.import_batch([blob], flags=A | LB_FLAG_EXPORT, lib_path=EMU)
    assert b.attribution_bytes(0) == want and b.export_updates(0) == oracle_doc([blob]).export_updates()
    assert b.timings()["attribution"] >= 0


def test_split_multibatch():
    blobs = [workloads.make_doc_history(600 + k, n_sites=2, n_ops=40)[0] for k in range(6)]
    b = loro_b200.import_batch(blobs, flags=A, lib_path=EMU, split=2)
    assert isinstance(b, loro_b200.api.MultiBatch)
    for k, blob in enumerate(blobs):
        assert b.attribution_bytes(k) == attribution_at(oracle_doc([blob]))
        parsed = b.attribution(k)
        assert all(isinstance(p, int) for runs in parsed.values() if isinstance(runs, list) for p, _, _ in runs)


def _traced_kernels(capfd):
    return [line.split()[2] for line in capfd.readouterr().err.splitlines() if line.startswith("simt_emu: launch ")]


def test_launch_count(monkeypatch, capfd):
    """without the flag nothing more is launched; with it three launches (count, scan, write) whatever the number of
    documents"""
    monkeypatch.setenv("LB_EMU_KTRACE", "1")
    for n in (1, 6):
        blobs = [workloads.make_doc_history(700 + k, n_sites=2, n_ops=50)[0] for k in range(n)]
        capfd.readouterr()
        plain = loro_b200.import_batch(blobs, lib_path=EMU)
        k0 = _traced_kernels(capfd)
        attr = loro_b200.import_batch(blobs, flags=A, lib_path=EMU)
        k1 = _traced_kernels(capfd)
        assert not any("k_attr" in k for k in k0)
        assert plain.timings()["kernel_launches"] == len(k0)
        assert attr.timings()["kernel_launches"] == len(k1) == len(k0) + 3
        assert sum("k_attr" in k for k in k1) == 2
