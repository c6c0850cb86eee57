"""lb_batch_export_json_updates on the emulated kernels: the engine's JSON text equals the reference's
(tests/json_updates_ref.cpp on the oracle) byte for byte, with and without peer compression, over random histories,
trees, import_batch groups, trimmed and pending changes, split changes, docsets and random version ranges; all requests
of a call cost one pass; errors per request and per call."""
import ctypes
import json
import os
import random
import subprocess

import pytest

import loro_b200
from loro_b200 import api
from oracle import OracleDoc
from tests import json_updates_checks as jc
from tests import workloads
from tests.test_engine_emu import _per_peer_blobs
from tests.test_export_emu import big_insert_documents

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")
INVALID_ARG, UNSUPPORTED = 1, 6


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def corpus():
    docs = [[workloads.make_doc_history(7100 + i, n_sites=2 + i % 3, n_ops=120 + 30 * i)[0]] for i in range(4)]
    docs += [[workloads.make_tree_history(80 + i, n_sites=2, n_base=10, n_ops=30, mixed=bool(i))[0]] for i in range(2)]
    big = big_insert_documents()
    docs += [[big[0]], [big[3]]]                            # changes split over several blocks
    e1, e2, n_partial = workloads.overlapping_update_blobs(9)
    assert n_partial > 0
    docs.append([e2, e1])                                   # trimmed changes
    docs.append([e1, e2, e1])                               # overlapping and repeated blobs
    docs.append([next(p for p in _per_peer_blobs(5400, n_sites=3, n_ops=100)[3] if OracleDoc(1).import_(p)["pending"])])
    return docs


def import_docs(docs, flags=api.LB_FLAG_EXPORT):
    blobs = [b for d in docs for b in d]
    ids = [k for k, d in enumerate(docs) for _ in d]
    return loro_b200.import_batch(blobs, doc_ids=ids, flags=flags, lib_path=EMU)


def test_corpus_matches_reference():
    docs = corpus()
    oracles = [jc.oracle_doc(d) for d in docs]
    batch = import_docs(docs)
    ranges = jc.seeded_ranges(11, len(docs), [o.oplog_vv() for o in oracles], per_doc=4)
    jc.compare_batch(batch, oracles, ranges)


def test_many_versions_one_pass(monkeypatch, capfd):
    docs = corpus()[:3]
    oracles = [jc.oracle_doc(d) for d in docs]
    batch = import_docs(docs)
    vv = oracles[0].oplog_vv()

    def launches(ranges):
        monkeypatch.setenv("LB_EMU_KTRACE", "1")
        capfd.readouterr()
        jc.compare_batch(batch, oracles, ranges, peer_compression=(True,))
        monkeypatch.delenv("LB_EMU_KTRACE")
        return sum(1 for line in capfd.readouterr().err.splitlines() if line.startswith("simt_emu: launch "))
    rng = random.Random(5)
    one = launches([(0, None, None)])
    many = launches([(0,) + jc.random_range(rng, vv) for _ in range(24)] + [(1, None, None), (2, {}, None)])
    assert one == many


def test_chunks(monkeypatch):
    docs = corpus()[:4]
    oracles = [jc.oracle_doc(d) for d in docs]
    batch = import_docs(docs)
    monkeypatch.setenv("LB_JSON_STAGE_CAP", "700")   # every request its own chunk, a few bigger than the cap
    jc.compare_batch(batch, oracles, jc.seeded_ranges(3, len(docs), [o.oplog_vv() for o in oracles], per_doc=2))


def test_messages_and_timestamps():
    a = OracleDoc(3)
    t = a.get_text("t")
    a.text_insert(t, 0, "héllo \"wörld\"\n")
    jc.commit_with(a, 1700000000, "first\tcommit")
    m = a.get_map("m")
    a.map_set(m, "k", 1.5)
    jc.commit_with(a, 1700000100, None)
    a.text_insert(t, 2, "🦜")
    jc.commit_with(a, 1700000200, "")
    blob = a.export_updates()
    oracles = [jc.oracle_doc([blob])]
    batch = import_docs([[blob]])
    jc.compare_batch(batch, oracles, [(0, None, None), (0, {3: 3}, None), (0, {3: 1}, {3: 16})])


def test_redact_known_answer():
    from tests.test_json_updates_oracle import REDACT_EXPECTED, redact_blob
    batch = import_docs([[redact_blob()]])
    assert json.dumps(json.loads(batch.export_json_updates(0)), indent=2, ensure_ascii=False) == REDACT_EXPECTED


def test_docset_and_read():
    rng = random.Random(4)
    s = loro_b200.DocSet(lib_path=EMU)
    ref = [OracleDoc(1) for _ in range(3)]
    per = [_per_peer_blobs(7400 + i, n_sites=3, n_ops=80)[3] for i in range(3)]
    last = None
    for r in range(3):
        blobs = [per[i][r % len(per[i])] for i in range(3)]
        for i in range(3):
            ref[i].import_(blobs[i])
        last = s.import_(blobs, doc_ids=[10, 11, 12], flags=api.LB_FLAG_EXPORT)
        ranges = [(i, None, None) for i in range(3)] + [(i,) + jc.random_range(rng, ref[i].oplog_vv()) for i in range(3)]
        jc.compare_batch(last, ref, ranges)
    read = s.read([12, 10])
    jc.compare_batch(read, [ref[2], ref[0]], [(0, None, None), (1, None, None), (1,) + jc.random_range(rng, ref[0].oplog_vv())])


def test_errors():
    good = workloads.make_doc_history(7500, n_sites=2, n_ops=60)[0]
    bad = bytearray(good)
    bad[-1] ^= 0xFF
    batch = import_docs([[good], [bytes(bad)]])
    out = batch.export_json_updates_many([(1, None, None), (0, None, None), (1, {}, {})])
    assert isinstance(out[0], api.EngineError) and out[0].status == INVALID_ARG
    assert out[1] == jc.export_json_updates(jc.oracle_doc([good]))
    assert isinstance(out[2], api.EngineError) and out[2].status == INVALID_ARG
    assert batch.export_json_updates_many([]) == []
    with pytest.raises(api.EngineError) as e:
        batch.export_json_updates_many([(0, None, None), (2, None, None)])
    assert e.value.status == INVALID_ARG
    # a null span pointer with a count fails the whole call
    arr = (api._JsonRequest * 1)()
    arr[0].doc, arr[0].start, arr[0].n_start = 0, None, 1
    h = ctypes.c_void_p()
    assert batch._L.lb_batch_export_json_updates(batch._h, arr, 1, ctypes.byref(h)) == INVALID_ARG
    plain = import_docs([[good]], flags=0)
    with pytest.raises(api.EngineError) as e:
        plain.export_json_updates(0)
    assert e.value.status == INVALID_ARG



def test_unsupported_next_to_supported():
    # a document the export phase does not cover (a MovableList op) answers LB_ERR_UNSUPPORTED without failing the
    # requests next to it
    from tests.test_export_many_emu import _bad_checksum_and_movable
    _, movable = _bad_checksum_and_movable()
    good = workloads.make_doc_history(7600, n_sites=2, n_ops=60)[0]
    batch = import_docs([[good], [movable]])
    out = batch.export_json_updates_many([(1, None, None), (0, None, None), (1, {}, {4: 3})])
    assert isinstance(out[0], api.EngineError) and out[0].status == UNSUPPORTED, out[0]
    assert isinstance(out[2], api.EngineError) and out[2].status == UNSUPPORTED, out[2]
    assert out[1] == jc.export_json_updates(jc.oracle_doc([good]))
