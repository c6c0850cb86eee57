"""lb_batch_export_updates and lb_docset_read on the emulated kernels: many export(updates(from)) requests in one call
answer byte for byte what one lb_doc_export_updates call per request answers, and what the oracle exports; the
launches of a call depend on the number of rounds only; the stored documents of a docset can be read and exported
without importing anything."""
import os
import random
import subprocess

import pytest

import loro_b200
from loro_b200 import api
from oracle import CT_MOVABLE, OracleDoc
from tests import workloads
from tests.docset_checks import _session
from tests.test_engine_emu import _per_peer_blobs
from tests.test_export_emu import big_insert_documents

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")
LACKING_PEER = 0xFEEDFACE
INVALID_ARG, UNSUPPORTED = 1, 6   # lb_status


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


@pytest.fixture
def launches(monkeypatch, capfd):
    """Switches the launch trace on; returns a function giving the kernels traced since its last call, by name."""
    monkeypatch.setenv("LB_EMU_KTRACE", "1")
    capfd.readouterr()

    def traced():
        return [line.split()[-1] for line in capfd.readouterr().err.splitlines() if line.startswith("simt_emu: launch ")]
    return traced


def corpus():
    """Documents as lists of blobs (several blobs = one import_batch group)"""
    docs = [[workloads.make_doc_history(5100 + i, n_sites=2 + i % 3, n_ops=140 + 30 * i)[0]] for i in range(4)]
    docs += [[workloads.make_tree_history(60 + i, n_sites=2, n_base=12, n_ops=40, mixed=bool(i))[0]] for i in range(2)]
    big = big_insert_documents()
    docs += [[big[0]], [big[3]]]                            # split changes and synthetic rows
    e1, e2, n_partial = workloads.overlapping_update_blobs(7)
    assert n_partial > 0
    docs.append([e2, e1])                                   # trimmed changes
    # one peer's changes alone, some of them depending on the other peers': pending changes
    docs.append([next(p for p in _per_peer_blobs(5300, n_sites=3, n_ops=120)[3] if OracleDoc(1).import_(p)["pending"])])
    return docs


def import_corpus(docs):
    blobs = [b for d in docs for b in d]
    ids = [k for k, d in enumerate(docs) for _ in d]
    return loro_b200.import_batch(blobs, doc_ids=ids, flags=api.LB_FLAG_EXPORT, lib_path=EMU)


def oracle_docs(docs):
    refs = []
    for d in docs:
        ref = OracleDoc(0xABCDEF)
        ref.import_batch(d)
        refs.append(ref)
    return refs


def versions_of(vv, rnd):
    """the oplog vv (header-only blob), {p: 1} (cut inside the first op), a lacking peer, counters past the vv, the
    empty version (None and {}), and random versions"""
    out = [dict(vv), {p: 1 for p in vv}, {LACKING_PEER: 3}, {p: c + 7 for p, c in vv.items()}, None, {}]
    out += [{p: rnd.randint(0, c) for p, c in vv.items() if rnd.random() < 0.8} for _ in range(2)]
    first = min(vv)
    out.append({first: vv[first] // 2, LACKING_PEER: 5})
    return out


def parity_requests(refs, seed):
    rnd = random.Random(seed)
    reqs = []
    for i, ref in enumerate(refs):
        vs = versions_of(ref.oplog_vv(), rnd)
        reqs += [(i, v) for v in (vs if i % 2 == 0 else rnd.sample(vs, 3))]   # some documents at many versions
    reqs += rnd.sample(reqs, 8)                                                 # duplicates
    rnd.shuffle(reqs)
    return reqs


def check_parity(batch, refs, reqs, docs):
    got = batch.export_updates_many(reqs)
    fresh = import_corpus(docs)
    for k, ((i, frm), g) in enumerate(zip(reqs, got)):
        want = refs[i].export_updates(frm)
        assert g == want, (k, i, frm, len(g), len(want))
        assert fresh.export_updates(i, frm) == want, (k, i, frm)
    return got


def test_many_requests_equal_single_calls_and_the_oracle():
    docs = corpus()
    refs = oracle_docs(docs)
    batch = import_corpus(docs)
    assert batch.status(len(docs) - 1).pending is not None
    check_parity(batch, refs, parity_requests(refs, 1), docs)


def test_many_requests_through_the_retry_encode(monkeypatch):
    """small staging slots: the blocks of many documents outgrow them in one round and are encoded again"""
    docs = corpus()
    refs = oracle_docs(docs)
    batch = import_corpus(docs)
    monkeypatch.setenv("LB_EXPORT_STAGE_CAP", "24")
    check_parity(batch, refs, parity_requests(refs, 2), docs)


def _bad_checksum_and_movable():
    blob = workloads.make_doc_history(4200, n_sites=2, n_ops=60)[0]
    bad = blob[:30] + bytes([blob[30] ^ 1]) + blob[31:]
    m = OracleDoc(4)
    mt = m.get_text("text")
    m.text_insert(mt, 0, "abc")
    m.commit()
    m.list_insert(m.container("mlist", CT_MOVABLE), 0, 1)
    m.commit()
    return bad, m.export_updates()


def test_failed_and_uncovered_documents_fail_their_requests_only():
    bad, movable = _bad_checksum_and_movable()
    good = [workloads.make_doc_history(4300 + i, n_sites=2, n_ops=80)[0] for i in range(2)]
    batch = loro_b200.import_batch([good[0], bad, movable, good[1]], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    assert [batch.status(i).code for i in range(4)] == [0, 2, 5, 0]
    refs = oracle_docs([[good[0]], [], [], [good[1]]])
    reqs = [(1, {1: 2}), (0, {p: 1 for p in refs[0].oplog_vv()}), (2, None), (3, None), (1, None), (2, {4: 1}),
            (3, {p: 2 for p in refs[3].oplog_vv()})]
    got = batch.export_updates_many(reqs)
    for (i, frm), g in zip(reqs, got):
        if i in (1, 2):
            want = INVALID_ARG if i == 1 else UNSUPPORTED
            assert isinstance(g, api.EngineError) and g.status == want, (i, frm, g)
            with pytest.raises(api.EngineError) as e:
                batch.export_updates(i, frm)
            assert e.value.status == want
        else:
            assert g == refs[i].export_updates(frm) == batch.export_updates(i, frm), (i, frm)


def test_whole_call_errors_launch_nothing(launches):
    blob = workloads.make_doc_history(4400, n_sites=2, n_ops=60)[0]
    batch = loro_b200.import_batch([blob], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    plain = loro_b200.import_batch([blob], lib_path=EMU)
    at = loro_b200.import_batch_at([blob], {0: []}, lib_path=EMU)
    launches()
    n0 = batch.timings()["kernel_launches"]
    for b, reqs in ((batch, [(0, None), (1, None)]), (plain, [(0, {1: 1})]), (at, [(0, None)])):
        with pytest.raises(api.EngineError) as e:
            b.export_updates_many(reqs)
        assert e.value.status == INVALID_ARG
    L = batch._L
    req = (api._ExportRequest * 1)()
    req[0].doc = 0
    req[0].n_from = 2                                       # from is NULL
    h = api.ctypes.c_void_p()
    assert L.lb_batch_export_updates(batch._h, req, 1, api.ctypes.byref(h)) == INVALID_ARG
    assert launches() == [] and batch.timings()["kernel_launches"] == n0
    assert batch.export_updates_many([]) == []


def launch_docs():
    """documents with something to export from {p: 1} in every one"""
    return [workloads.make_doc_history(4500 + i, n_sites=2 + i % 2, n_ops=90)[0] for i in range(5)]


def test_launches_depend_on_rounds_not_documents(launches, monkeypatch):
    monkeypatch.setenv("LB_EXPORT_STAGE_CAP", "0")          # every block takes the retry encode: one more launch per round
    blobs = launch_docs()
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    vvs = [batch.oplog_vv(i) for i in range(len(blobs))]
    cut = [{p: 1 for p in vv} for vv in vvs]
    launches()
    n0 = batch.timings()["kernel_launches"]

    def traced_call(reqs):
        before = batch.timings()["kernel_launches"]
        out = batch.export_updates_many(reqs)
        t = launches()
        assert batch.timings()["kernel_launches"] - before == len(t)
        assert all(not isinstance(o, api.EngineError) for o in out)
        return t

    one = traced_call([(2, cut[2])])
    every = traced_call([(i, cut[i]) for i in range(len(blobs))])
    assert one.count("k_exp_encode<1>") + one.count("k_exp_encode<0>") == 2
    assert len(one) == len(every) > 0
    # three distinct versions of one document: three rounds, as many launches as three one-request calls
    vs = [cut[0], {p: c // 2 for p, c in vvs[0].items()}, {p: max(1, c - 3) for p, c in vvs[0].items()}]
    three = traced_call([(0, v) for v in vs])
    single = sum(len(traced_call([(0, v)])) for v in vs)
    assert len(three) == single
    # identical requests: one round
    assert len(traced_call([(1, cut[1])] * 4)) == len(one)
    # everything asked for: the import-time export, no launch
    assert traced_call([(3, None), (3, {}), (3, {LACKING_PEER: 9}), (3, {p: 0 for p in vvs[3]})]) == []
    assert batch.timings()["kernel_launches"] > n0


def test_nothing_else_changes():
    docs = corpus()
    refs = oracle_docs(docs)
    batch = import_corpus(docs)
    before = [(batch.export_updates(i), batch.json_bytes(i), batch.oplog_vv(i)) for i in range(len(docs))]
    batch.export_updates_many(parity_requests(refs, 3))
    for i in range(len(docs)):
        assert (batch.export_updates(i), batch.json_bytes(i), batch.oplog_vv(i)) == before[i], i
        frm = {p: c // 3 for p, c in refs[i].oplog_vv().items()}
        assert batch.export_updates(i, frm) == refs[i].export_updates(frm), i


def test_results_outlive_the_batch():
    blob = workloads.make_doc_history(4600, n_sites=3, n_ops=100)[0]
    ref = OracleDoc(1)
    ref.import_(blob)
    frm = {p: 2 for p in ref.oplog_vv()}
    batch = loro_b200.import_batch([blob], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    L = batch._L
    req = (api._ExportRequest * 2)()
    spans, k = api._vv_spans(frm)
    req[0].doc, req[0].from_, req[0].n_from = 0, spans, k
    req[1].doc = 0
    h = api.ctypes.c_void_p()
    assert L.lb_batch_export_updates(batch._h, req, 2, api.ctypes.byref(h)) == 0
    batch.close()
    for j, want in enumerate((ref.export_updates(frm), ref.export_updates())):
        p, n = api.ctypes.c_void_p(), api.ctypes.c_size_t()
        assert L.lb_exports_get(h, j, api.ctypes.byref(p), api.ctypes.byref(n)) == 0
        assert api.ctypes.string_at(p.value, n.value) == want
    assert L.lb_exports_get(h, 2, api.ctypes.byref(p), api.ctypes.byref(n)) == INVALID_ARG
    L.lb_exports_free(h)


def test_split_batch_equals_the_unsplit_one():
    blobs = [workloads.make_doc_history(4700 + i, n_sites=2 + i % 3, n_ops=100)[0] for i in range(6)]
    whole = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU, split=1)
    split = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU, split=2)
    assert isinstance(split, api.MultiBatch)
    rnd = random.Random(5)
    reqs = [(i, v) for i in range(len(blobs)) for v in versions_of(whole.oplog_vv(i), rnd)[:5]]
    rnd.shuffle(reqs)
    assert split.export_updates_many(reqs) == whole.export_updates_many(reqs)


# ------------------------------------------------------------------ lb_docset_read
def check_docset_read(lib_path=None, n_docs=4, rounds=4, edits=8, seed=11):
    """after several lb_docset_import calls, DocSet.read answers what the batch of each document's last import answered,
    exports like the oracle, reads an unknown id as an empty document and leaves the set as it was"""
    rnd = random.Random(seed)
    streams = {600 + d: _session(40 + seed + d, 2 + d % 2, rounds, edits) for d in range(n_docs)}
    ds = loro_b200.DocSet(lib_path=lib_path)
    refs = {d: OracleDoc(0xD0C) for d in streams}
    last = {}
    cursors = dict.fromkeys(streams, 0)
    while any(cursors[d] < len(s) for d, s in streams.items()):
        blobs, ids = [], []
        for d, s in streams.items():
            if cursors[d] < len(s) and rnd.random() < 0.7:
                take = s[cursors[d]:cursors[d] + rnd.randint(1, 2)]
                cursors[d] += len(take)
                refs[d].import_batch(take)
                blobs += take
                ids += [d] * len(take)
        if not blobs:
            continue
        b = ds.import_(blobs, ids)
        for slot, d in enumerate(dict.fromkeys(ids)):
            last[d] = (b.json_bytes(slot), b.oplog_vv(slot), b.oplog_frontiers(slot), b.export_updates(slot))
        b.close()
    n_docs, stored = ds.n_docs, ds.stored_bytes
    order = list(streams)
    rnd.shuffle(order)
    order.insert(1, 12345)                                  # never seen
    r = ds.read(order)
    assert r.n_docs == len(order)
    for slot, d in enumerate(order):
        st = r.status(slot)
        assert st.code == 0 and st.success == {} and st.pending is None, (d, st)
        if d not in streams:
            assert r.json_bytes(slot) == b"{}" and r.oplog_vv(slot) == {} and r.oplog_frontiers(slot) == []
            assert r.export_updates(slot) == OracleDoc(1).export_updates()
            continue
        got = (r.json_bytes(slot), r.oplog_vv(slot), r.oplog_frontiers(slot), r.export_updates(slot))
        assert got == last[d], d
        assert got[0] == refs[d].json_text() and got[3] == refs[d].export_updates()
    reqs = []
    for slot, d in enumerate(order):
        if d in streams:
            reqs += [(slot, v) for v in versions_of(refs[d].oplog_vv(), rnd)[:6]]
    rnd.shuffle(reqs)
    for (slot, frm), g in zip(reqs, r.export_updates_many(reqs)):
        assert g == refs[order[slot]].export_updates(frm), (slot, frm)
    r.close()
    assert (ds.n_docs, ds.stored_bytes) == (n_docs, stored)
    # the read left the set as it was: one more update imports exactly as it would have
    a = OracleDoc(77)
    a.text_insert(a.get_text("text"), 0, "late")
    a.commit()
    extra = a.export_updates()
    b = ds.import_([extra], [601])
    st = refs[601].import_(extra)
    assert b.status(0).success == st["success"] and b.json_bytes(0) == refs[601].json_text()
    assert b.export_updates(0) == refs[601].export_updates()
    ds.close()


def test_docset_read_answers_for_the_stored_documents():
    check_docset_read(lib_path=EMU)


def test_docset_read_flags_and_errors():
    ds = loro_b200.DocSet(lib_path=EMU)
    blob = workloads.make_doc_history(4800, n_sites=2, n_ops=60)[0]
    ds.import_([blob], [5]).close()
    r = ds.read([5], flags=api.LB_FLAG_NO_JSON)
    with pytest.raises(api.EngineError):
        r.json_bytes(0)
    ref = OracleDoc(1)
    ref.import_(blob)
    assert r.export_updates(0) == ref.export_updates()
    for ids, flags in (([5, 5], 0), ([5], api.LB_FLAG_COMPACT)):
        with pytest.raises(api.EngineError) as e:
            ds.read(ids, flags=flags)
        assert e.value.status == INVALID_ARG
    assert ds.read([]).n_docs == 0
    ds.close()
