"""Cursors on the H100 (the CUDA build): a batch of full-size C3 documents with cursors on every document in one call,
C5 (tree containers refused, the text in them answered), the automerge trace with cursors on many deleted characters,
and one C3 document with thousands of cursors in one call -- field for field against the reference
(tests/cursor_ref.cpp)."""
import gzip
import os
import random

import pytest

import loro_b200
from loro_b200.api import LB_CURSOR_ID_NOT_FOUND, LB_FLAG_ATTRIBUTION, LB_FLAG_CURSORS

from .checkout_checks import oracle_doc
from .cursor_checks import cursor_pos_ref, sample_cursors, seq_containers

pytestmark = pytest.mark.gpu
F = LB_FLAG_CURSORS


def _engine_cursors(b, i, rnd, k):
    """k cursors on document i of b over the Text / List containers its attribution lists"""
    cids = [c for c in b.attribution(i) if c.endswith((":Text", ":List"))] or ["cid:root-absent:Text"]
    return sample_cursors(rnd, cids, b.oplog_vv(i), k)


def test_full_size_c3_batch_every_document_in_one_call():
    from loro_b200.workload import C3Batch
    blobs = C3Batch(256, n_ops=10000, threads=8).blobs()
    b = loro_b200.import_batch(blobs, flags=F | LB_FLAG_ATTRIBUTION)
    rnd = random.Random(31)
    per_doc = {i: _engine_cursors(b, i, rnd, 64) for i in range(len(blobs))}
    reqs = [(i,) + c for i in per_doc for c in per_doc[i]]
    got = b.cursor_pos(reqs)
    assert all(s in (0, LB_CURSOR_ID_NOT_FOUND) for s, _, _, _ in got)
    assert sum(u is not None for _, _, _, u in got) > len(got) // 20      # many deleted targets
    for i in rnd.sample(range(len(blobs)), 12):
        lo = 64 * i
        assert got[lo:lo + 64] == cursor_pos_ref(oracle_doc([blobs[i]]), per_doc[i]), i


def test_c5_tree_containers_are_refused_and_text_answers():
    from loro_b200.workload import C5Batch
    blobs = C5Batch(24, threads=8).blobs()
    b = loro_b200.import_batch(blobs, flags=F | LB_FLAG_ATTRIBUTION)
    rnd = random.Random(32)
    for i in range(0, len(blobs), 6):
        doc = oracle_doc([blobs[i]])
        trees = [c for c in b.attribution(i) if c.endswith(":Tree")]
        assert trees
        got = b.cursor_pos([(i, c, None, 0) for c in trees])
        assert all(s == 1 for s, _, _, _ in got)
        seqs = list(seq_containers(doc)) + ["cid:root-absent:Text"]
        cs = sample_cursors(rnd, seqs, doc.oplog_vv(), 200)
        assert b.cursor_pos([(i,) + c for c in cs]) == cursor_pos_ref(doc, cs), i


def test_automerge_trace_cursors_on_deleted_characters(golden_dir):
    blob = gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read()
    b = loro_b200.import_batch([blob], flags=F)
    doc = oracle_doc([blob])
    rnd = random.Random(33)
    cs = sample_cursors(rnd, list(seq_containers(doc)), doc.oplog_vv(), 4000)
    got = b.cursor_pos([(0,) + c for c in cs])
    assert got == cursor_pos_ref(doc, cs)
    assert sum(u is not None for _, _, _, u in got) > 500


def test_one_c3_document_thousands_of_cursors_in_one_call():
    from loro_b200.workload import C3Batch
    blob = C3Batch(1, n_ops=10000, threads=8).blob(0)
    b = loro_b200.import_batch([blob], flags=F)
    doc = oracle_doc([blob])
    rnd = random.Random(34)
    cs = sample_cursors(rnd, list(seq_containers(doc)) + ["cid:root-absent:List"], doc.oplog_vv(), 8000)
    assert b.cursor_pos([(0,) + c for c in cs]) == cursor_pos_ref(doc, cs)
