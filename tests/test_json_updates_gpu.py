"""lb_batch_export_json_updates on the H100 (the CUDA build): the emulated suite's corpus against the reference byte for
byte; full-size C3 and C5 documents, a sample of them against the reference and every document of a 4,096-document C3
call against the invariants; one C3 document at 64 version ranges in one call."""
import random

import pytest

import loro_b200
from loro_b200 import api
from oracle import OracleDoc

from . import json_updates_checks as jc
from .test_json_updates_emu import corpus

pytestmark = pytest.mark.gpu


def _import(docs):
    blobs = [b for d in docs for b in d]
    ids = [k for k, d in enumerate(docs) for _ in d]
    return loro_b200.import_batch(blobs, doc_ids=ids, flags=api.LB_FLAG_EXPORT)


def test_corpus_matches_reference():
    docs = corpus()
    oracles = [jc.oracle_doc(d) for d in docs]
    batch = _import(docs)
    jc.compare_batch(batch, oracles, jc.seeded_ranges(21, len(docs), [o.oplog_vv() for o in oracles], per_doc=6))


def test_c3_and_c5_full_size():
    from loro_b200.workload import C3Batch, C5Batch
    c3 = C3Batch(16, n_ops=10000, threads=8).blobs()
    c5 = C5Batch(8).blobs()
    blobs = c3 + c5
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON)
    rng = random.Random(7)
    sample = [0, 1, len(c3), len(c3) + 1]
    oracles = {}
    ranges = []
    for i in sample:
        oracles[i] = OracleDoc(0xABCDEF)
        oracles[i].import_(blobs[i])
        vv = oracles[i].oplog_vv()
        ranges += [(i, None, None), (i,) + jc.random_range(rng, vv)]
    jc.compare_batch(batch, oracles, ranges)
    # one C3 document at 64 version ranges in one call
    vv = oracles[0].oplog_vv()
    many = [(0,) + jc.random_range(rng, vv) for _ in range(64)]
    jc.compare_batch(batch, oracles, many, peer_compression=(True,))


def test_4096_c3_documents_invariants():
    from loro_b200.workload import C3Batch
    blobs = C3Batch(4096, n_ops=10000, threads=16).blobs()
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON)
    got = batch.export_json_updates_many([(i, None, None) for i in range(len(blobs))])
    for i, g in enumerate(got):
        assert isinstance(g, str), (i, g)
        vv = batch.oplog_vv(i)
        jc.check_invariants(g, {}, vv, vv)
