"""Attribution on the H100 (the CUDA build): full-size C3 and C5 documents, one C3 document at 256 versions in one
checkout, and the automerge trace's single long text, byte for byte against the reference (tests/attribution_ref.cpp)."""
import gzip
import os
import random

import pytest

import loro_b200
from loro_b200.api import LB_FLAG_ATTRIBUTION

from . import workloads
from .attribution_checks import attribution_at
from .checkout_checks import applied_ids, oracle_doc, random_frontiers

pytestmark = pytest.mark.gpu
A = LB_FLAG_ATTRIBUTION


def _check_latest(blobs):
    b = loro_b200.import_batch(blobs, flags=A)
    for k, blob in enumerate(blobs):
        assert b.status(k).code == 0, k
        assert b.attribution_bytes(k) == attribution_at(oracle_doc([blob])), k
    return b


def test_random_histories_and_trees():
    rnd = random.Random(21)
    blobs = [workloads.make_doc_history(8000 + k, n_sites=rnd.randint(1, 5), n_ops=rnd.randint(60, 400))[0]
             for k in range(64)]
    blobs += [workloads.make_tree_history(900 + k, n_sites=3, n_base=40, n_ops=150, mixed=k % 3 == 0)[0] for k in range(16)]
    _check_latest(blobs)


def test_full_size_c3_documents():
    from loro_b200.workload import C3Batch
    _check_latest(C3Batch(24, n_ops=10000, threads=8).blobs())


def test_full_size_c5_documents():
    from loro_b200.workload import C5Batch
    _check_latest(C5Batch(24, threads=8).blobs())


def test_one_c3_document_at_256_versions_in_one_checkout():
    from loro_b200.workload import C3Batch
    blob = C3Batch(1, n_ops=10000, threads=8).blob(0)
    o = oracle_doc([blob])
    ids = applied_ids(o)
    rnd = random.Random(22)
    versions = [[ids[(k * len(ids)) // 256]] if k % 2 else random_frontiers(rnd, o, max_ids=2) for k in range(256)]
    ds = loro_b200.DocSet()
    ds.import_([blob], [3])
    r = ds.checkout([(3, f) for f in versions], flags=A)
    assert r.n_docs == 256
    for k, f in enumerate(versions):
        assert r.status(k).code == 0, f
        assert r.attribution_bytes(k) == attribution_at(o, f), (k, f)


def test_automerge_trace(golden_dir):
    """one Text of ~10^5 characters written in ~2.6 * 10^5 edits: the runs are printed by all lanes of the warp"""
    blob = gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read()
    b = _check_latest([blob])
    runs = next(iter(b.attribution(0).values()))
    assert len(runs) > 1000
