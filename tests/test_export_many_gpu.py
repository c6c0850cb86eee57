"""lb_batch_export_updates and lb_docset_read on the H100 (the CUDA build): full-size C3 documents and C5 tree documents at
random versions in one call, equal to one lb_doc_export_updates call per request and to the oracle; DocSet.read on
docset streams of the GPU tests' size."""
import random

import pytest

import loro_b200
from loro_b200 import api
from oracle import OracleDoc

from .test_export_many_emu import check_docset_read

pytestmark = pytest.mark.gpu


def test_c3_and_c5_documents_at_random_versions_in_one_call():
    from loro_b200.workload import C3Batch, C5Batch
    c3 = C3Batch(64, n_ops=10000, threads=8).blobs()
    c5 = C5Batch(24).blobs()
    blobs = c3 + c5
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON, split=1)
    rnd = random.Random(3)
    reqs = []
    for i in range(len(blobs)):
        vv = batch.oplog_vv(i)
        for _ in range(1 if i % 3 else 3):                  # every third document at three versions: three rounds
            reqs.append((i, {p: rnd.randint(0, c) for p, c in vv.items()}))
    rnd.shuffle(reqs)
    got = batch.export_updates_many(reqs)
    for (i, frm), g in zip(reqs, got):
        assert not isinstance(g, api.EngineError), (i, g)
        assert g == batch.export_updates(i, frm), (i, frm)
    checked = set()
    for (i, frm), g in zip(reqs, got):
        group = i < len(c3)
        if sum(1 for j in checked if (j < len(c3)) == group) >= 8 or i in checked:
            continue
        ref = OracleDoc(0xABCDEF)
        ref.import_(blobs[i])
        assert g == ref.export_updates(frm), (i, frm)
        checked.add(i)
    assert len(checked) == 16


@pytest.mark.parametrize("seed", range(2))
def test_docset_read_of_stored_documents(seed):
    check_docset_read(n_docs=12, rounds=8, edits=16, seed=seed)
