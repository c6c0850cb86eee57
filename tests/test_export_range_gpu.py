"""lb_batch_export_updates_in_range on the H100 (the CUDA build): full-size C3 documents and C5 tree documents at random
span sets in one call, equal to one call per request and to the reference's UpdatesInRange export."""
import random

import pytest

import loro_b200
from loro_b200 import api
from oracle import OracleDoc

from .range_export_checks import Refused, export_in_range, span_sets

pytestmark = pytest.mark.gpu


def test_c3_and_c5_documents_at_random_ranges_in_one_call():
    from loro_b200.workload import C3Batch, C5Batch
    c3 = C3Batch(64, n_ops=10000, threads=8).blobs()
    c5 = C5Batch(24).blobs()
    blobs = c3 + c5
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON, split=1)
    rnd = random.Random(4)
    reqs = []
    for i in range(len(blobs)):
        sets = span_sets(batch.oplog_vv(i), rnd)
        reqs += [(i, s) for s in rnd.sample(sets, 3 if i % 3 == 0 else 1)]   # every third document: three rounds
    rnd.shuffle(reqs)
    got = batch.export_updates_in_range_many(reqs)
    checked = set()
    for (i, spans), g in zip(reqs, got):
        single = batch.export_updates_in_range_many([(i, spans)])[0]
        assert type(g) is type(single), (i, spans, g, single)
        if not isinstance(g, api.EngineError):
            assert g == single, (i, spans)
        group = i < len(c3)
        if sum(1 for j in checked if (j < len(c3)) == group) >= 8 or i in checked:
            continue
        ref = OracleDoc(0xABCDEF)
        ref.import_(blobs[i])
        try:
            want = export_in_range(ref, spans)
        except Refused:
            assert isinstance(g, api.EngineError) and g.status == 1, (i, spans, g)
        else:
            assert g == want, (i, spans)
        checked.add(i)
    assert len(checked) == 16
