"""lb_batch_export_updates_in_range on the emulated kernels: every answer equals the reference's UpdatesInRange export
(tests/range_export_ref.cpp) byte for byte, many-request calls agree with single calls, refused and failed requests
leave the rest of the call alone, and the launches of a call depend on its number of rounds only."""
import random

import pytest

import loro_b200
from loro_b200 import api
from oracle import OracleDoc
from tests import workloads
from tests.range_export_checks import (BATCH_STATUS_SPANS, LACKING_PEER, Refused, check_requests, export_in_range,
                                       hello_docs, random_requests, till_spans)
from tests.test_export_many_emu import (EMU, INVALID_ARG, UNSUPPORTED, _bad_checksum_and_movable, build_emu,  # noqa: F401
                                        corpus, import_corpus, launch_docs, launches, oracle_docs)


def test_range_requests_equal_the_reference_and_single_calls():
    docs = corpus()
    refs = oracle_docs(docs)
    batch = import_corpus(docs)
    check_requests(batch, refs, random_requests(refs, 1))


def test_range_requests_through_the_retry_encode(monkeypatch):
    """small staging slots: the blocks of many documents outgrow them in one round and are encoded again"""
    docs = corpus()
    refs = oracle_docs(docs)
    batch = import_corpus(docs)
    monkeypatch.setenv("LB_EXPORT_STAGE_CAP", "24")
    check_requests(batch, refs, random_requests(refs, 2, per_doc=8), single=False)


def test_whole_and_from_spans_equal_the_other_exports():
    """one span [0, vv) per peer is all_updates; one span [from, vv) per peer is updates(from)"""
    docs = corpus()
    refs = oracle_docs(docs)
    batch = import_corpus(docs)
    rnd = random.Random(3)
    for i, ref in enumerate(refs):
        vv = ref.oplog_vv()
        assert batch.export_updates_till(i, vv) == batch.export_updates(i) == ref.export_updates(), i
        frm = {p: rnd.randint(0, c) for p, c in vv.items()}
        want = ref.export_updates(frm)
        assert batch.export_updates_in_range(i, [(p, frm[p], c) for p, c in vv.items()]) == want, (i, frm)
        assert export_in_range(ref, [(p, frm[p], c) for p, c in vv.items()]) == want, (i, frm)


def test_import_batch_status_on_engine_range_blobs():
    """loro_import_batch_status on range blobs the engine made, imported by the engine as import_batch groups into one
    stored document: the reference's statuses and text"""
    refs = hello_docs()
    src = loro_b200.import_batch([d.export_updates() for d in refs], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    reqs = [(spans[0][0] - 1, spans) for spans in BATCH_STATUS_SPANS]
    b11, b12, b13, b21, b22, b23 = src.export_updates_in_range_many(reqs)
    for (i, spans), g in zip(reqs, (b11, b12, b13, b21, b22, b23)):
        assert g == export_in_range(refs[i], spans), spans
    ds = loro_b200.DocSet(lib_path=EMU)
    first = ds.import_([b11, b13, b21, b23], [9] * 4)
    st = first.status(0)
    assert st.success == {1: (0, 5), 2: (0, 5)} and st.pending == {1: (6, 12), 2: (6, 12)}
    second = ds.import_([b12, b22], [9, 9])
    st = second.status(0)
    assert st.success == {1: (5, 12), 2: (5, 12)} and st.pending is None
    assert second.get_deep_value(0) == {"text": "Hello world!Hello world!"}
    ds.close()


def test_refused_and_failed_requests_leave_the_rest():
    bad, movable = _bad_checksum_and_movable()
    good = [workloads.make_doc_history(4300 + i, n_sites=2, n_ops=80)[0] for i in range(2)]
    batch = loro_b200.import_batch([good[0], bad, movable, good[1]], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    refs = oracle_docs([[good[0]], [], [], [good[1]]])
    p0 = min(refs[0].oplog_vv())
    c0 = refs[0].oplog_vv()[p0]
    gap = [(p0, 0, 2), (p0, 4, c0)]
    overlap = [(p0, 0, 4), (p0, 2, c0)]
    reqs = [(0, gap), (1, [(1, 0, 2)]), (3, till_spans(refs[3].oplog_vv())), (0, overlap), (2, [(4, 0, 1)]),
            (0, [(p0, 4, c0), (p0, 0, 2)])]
    got = batch.export_updates_in_range_many(reqs)
    for (i, spans), g in zip(reqs, got):
        if i in (1, 2):
            assert isinstance(g, api.EngineError) and g.status == (INVALID_ARG if i == 1 else UNSUPPORTED), (i, g)
            continue
        try:
            want = export_in_range(refs[i], spans)
        except Refused:
            assert isinstance(g, api.EngineError) and g.status == INVALID_ARG, (i, spans, g)
            with pytest.raises(api.EngineError):
                batch.export_updates_in_range(i, spans)
            continue
        assert g == want, (i, spans)
    assert all(isinstance(got[k], api.EngineError) for k in (0, 3))
    assert not isinstance(got[5], api.EngineError)


def test_whole_call_errors_launch_nothing(launches):
    blob = workloads.make_doc_history(4400, n_sites=2, n_ops=60)[0]
    batch = loro_b200.import_batch([blob], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    plain = loro_b200.import_batch([blob], lib_path=EMU)
    launches()
    n0 = batch.timings()["kernel_launches"]
    for b, reqs in ((batch, [(0, []), (1, [])]), (plain, [(0, [(1, 0, 1)])])):
        with pytest.raises(api.EngineError) as e:
            b.export_updates_in_range_many(reqs)
        assert e.value.status == INVALID_ARG
    req = (api._RangeRequest * 1)()
    req[0].doc = 0
    req[0].n_spans = 2                                      # spans is NULL
    h = api.ctypes.c_void_p()
    assert batch._L.lb_batch_export_updates_in_range(batch._h, req, 1, api.ctypes.byref(h)) == INVALID_ARG
    assert launches() == [] and batch.timings()["kernel_launches"] == n0
    assert batch.export_updates_in_range_many([]) == []


def test_launches_depend_on_rounds_not_documents_or_spans(launches, monkeypatch):
    monkeypatch.setenv("LB_EXPORT_STAGE_CAP", "0")          # every block takes the retry encode: one more launch per round
    blobs = launch_docs()
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    vvs = [batch.oplog_vv(i) for i in range(len(blobs))]
    launches()

    def traced(reqs):
        out = batch.export_updates_in_range_many(reqs)
        assert all(not isinstance(o, api.EngineError) for o in out)
        return launches()

    def two_sided(vv, k):
        return [(p, min(k, c), max(c - k, min(k, c))) for p, c in vv.items()]

    one = traced([(2, two_sided(vvs[2], 1))])
    # spans that end inside a change take the encoder build with end cuts; the others keep the build without them
    assert one.count("k_exp_encode_cut<0>") == 2 and "k_exp_encode<0>" not in one
    from_shaped = traced([(2, [(p, 1, c) for p, c in vvs[2].items()])])
    assert from_shaped.count("k_exp_encode<0>") == 2 and "k_exp_encode_cut<0>" not in from_shaped
    every = traced([(i, two_sided(vvs[i], 1)) for i in range(len(blobs))])
    assert len(one) == len(every) > 0
    many_spans = [(p, a, a + 1) for p, c in vvs[0].items() for a in range(c - 1, -1, -1)]   # one span per atom
    assert len(traced([(0, many_spans)])) == len(one)
    sets = [two_sided(vvs[0], k) for k in (1, 2, 3)]
    assert len(traced([(0, s) for s in sets])) == 3 * len(one)
    assert len(traced([(1, two_sided(vvs[1], 2))] * 4)) == len(one)
    # everything asked for: the import-time export, no launch
    assert traced([(3, till_spans(vvs[3])), (3, till_spans(vvs[3]) + [(LACKING_PEER, 0, 4)])]) == []
