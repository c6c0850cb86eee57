"""Checkout on the H100 (the CUDA build): the checks of tests/test_checkout_emu.py at GPU sizes, full-size C3 documents at
random versions, and one C3 document at 256 versions in one call, against the oracle's capped replay."""
import random

import pytest

import loro_b200
from oracle import OracleDoc

from . import workloads
from .checkout_checks import (FRONTIERS_NOT_FOUND, applied_ids, check_import_batch_at, interesting_ids, json_at,
                              oracle_doc, random_frontiers)

pytestmark = pytest.mark.gpu


def test_random_histories_at_random_ids():
    rnd = random.Random(11)
    groups, requests = [], {}
    for k in range(96):
        blob, _, _, _ = workloads.make_doc_history(5000 + k, n_sites=rnd.randint(1, 5), n_ops=rnd.randint(60, 400))
        groups.append([blob])
        o = oracle_doc([blob])
        inside = interesting_ids(blob)
        pick = k % 4
        if pick == 0 and inside:
            requests[k] = [rnd.choice(inside)]
        elif pick == 1:
            requests[k] = random_frontiers(rnd, o, max_ids=5)
        elif pick == 2:
            requests[k] = [rnd.choice(applied_ids(o))]
        elif k % 8 == 3:
            requests[k] = []
    check_import_batch_at(groups, requests)


def test_tree_histories():
    rnd = random.Random(12)
    groups, requests = [], {}
    for k in range(24):
        blob, _, _, _ = workloads.make_tree_history(700 + k, n_sites=3, n_base=40, n_ops=150, mixed=k % 3 == 0)
        groups.append([blob])
        requests[k] = random_frontiers(rnd, oracle_doc([blob]), max_ids=3)
    check_import_batch_at(groups, requests)


def test_groups_with_overlapping_blobs_and_invalid_ids():
    rnd = random.Random(13)
    groups, requests, codes = [], {}, {}
    for k in range(8):
        e1, e2, _ = workloads.overlapping_update_blobs(20 + k)
        groups.append([e1, e2] if k % 2 else [e2, e1])
        requests[len(groups) - 1] = [rnd.choice(interesting_ids(e2) + applied_ids(oracle_doc(groups[-1])))]
    a = OracleDoc(1)
    t = a.get_text("text")
    a.text_insert(t, 0, "abc")
    a.commit()
    a.text_insert(t, 3, "def")
    a.commit()
    pend = a.export_updates({1: 3})
    for f in ([(1, 4)], [(99, 0)]):            # inside a pending change ; unknown peer
        groups.append([pend])
        requests[len(groups) - 1] = f
        codes[len(groups) - 1] = FRONTIERS_NOT_FOUND
    blob = workloads.make_doc_history(31, n_sites=2, n_ops=80)[0]
    vv = oracle_doc([blob]).oplog_vv()
    p0 = next(iter(vv))
    groups.append([blob])
    requests[len(groups) - 1] = [(p0, vv[p0])]   # a counter at the vv
    codes[len(groups) - 1] = FRONTIERS_NOT_FOUND
    check_import_batch_at(groups, requests, expect_codes=codes)


def test_full_size_c3_documents_at_random_versions():
    from loro_b200.workload import C3Batch
    gen = C3Batch(24, n_ops=10000, threads=8)
    blobs = gen.blobs()
    rnd = random.Random(14)
    requests = {}
    for k, blob in enumerate(blobs):
        o = oracle_doc([blob])
        requests[k] = [rnd.choice(interesting_ids(blob))] if k % 2 else random_frontiers(rnd, o, max_ids=3)
    check_import_batch_at([[b] for b in blobs], requests)


def test_one_c3_document_at_256_versions_in_one_call():
    from loro_b200.workload import C3Batch
    blob = C3Batch(1, n_ops=10000, threads=8).blob(0)
    o = oracle_doc([blob])
    ids = applied_ids(o)
    rnd = random.Random(15)
    versions = [[ids[(k * len(ids)) // 256]] if k % 2 else [rnd.choice(ids), rnd.choice(ids)] for k in range(256)]
    ds = loro_b200.DocSet()
    ds.import_([blob], [3])
    stored = ds.stored_bytes
    r = ds.checkout([(3, f) for f in versions])
    assert r.n_docs == 256
    for k, f in enumerate(versions):
        assert r.status(k).code == 0, f
        assert r.json_bytes(k) == json_at(o, f), (k, f)
    assert ds.stored_bytes == stored and ds.n_docs == 1


def test_docset_history_browsing():
    from .docset_checks import _session
    blobs = _session(8, n_sites=4, rounds=10, edits=24)
    ds = loro_b200.DocSet()
    ref = OracleDoc(9)
    seen = []
    for blob in blobs:
        r = ds.import_([blob], [4])
        ref.import_(blob)
        if ref.pending_count() == 0:
            seen.append(r.oplog_frontiers(0))
    stored, n = ds.stored_bytes, ds.n_docs
    r = ds.checkout([(4, f) for f in seen])
    for k, f in enumerate(seen):
        assert r.status(k).code == 0 and r.json_bytes(k) == json_at(ref, f), (k, f)
    assert ds.stored_bytes == stored and ds.n_docs == n
    last = workloads.make_doc_history(6, n_sites=2, n_ops=30)[0]
    r2 = ds.import_([last], [4])
    ref.import_(last)
    assert r2.json_bytes(0) == ref.json_text() and r2.export_updates(0) == ref.export_updates()
