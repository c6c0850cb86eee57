#!/usr/bin/env python3
"""export(ExportMode::UpdatesInRange / updates_till) for many documents in one lb_batch_export_updates_in_range call.

Leg (a): `--docs` documents of config C3's shape, imported with LB_FLAG_EXPORT | LB_FLAG_NO_JSON; every document at a
seeded random updates_till(vv) (one span [0, vv[p]) per peer), all in ONE call (one round).  Leg (b): the same
documents at seeded random two-sided ranges [a, b) per peer, one call.  Leg (c): ONE C3 document at `--sets` distinct
span sets in one call (one round each).  Each leg: host wall milliseconds of the call (it ends in a synchronise),
median of `--steps` after one warm-up, and the bytes it returns.  Prints one JSON line; the card and its power limit
are part of it.

  python scripts/bench_export_range.py [--docs 40000] [--ops 10000] [--steps 3] [--sets 64]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_export_many import card  # noqa: E402


def request_array(reqs):
    """[(doc, [(peer, start, end), ...]), ...] -> lb_range_request array (+ the span arrays it points into)"""
    from loro_b200 import api
    arr = (api._RangeRequest * max(len(reqs), 1))()
    keep = []
    for j, (doc, spans) in enumerate(reqs):
        sp = (api._IdSpan * max(len(spans), 1))()
        for k, (p, a, b) in enumerate(spans):
            sp[k].peer, sp[k].start, sp[k].end = p, a, b
        keep.append(sp)
        arr[j].doc, arr[j].spans, arr[j].n_spans = doc, sp, len(spans)
    return arr, keep


def timed(batch, reqs, steps):
    """median host ms of one lb_batch_export_updates_in_range call over `steps` after a warm-up, and its bytes"""
    import torch
    L = batch._L
    arr, keep = request_array(reqs)
    times, total = [], 0
    for step in range(steps + 1):
        torch.cuda.synchronize()
        h = ctypes.c_void_p()
        t0 = time.perf_counter()
        rc = L.lb_batch_export_updates_in_range(batch._h, arr, len(reqs), ctypes.byref(h))
        ms = (time.perf_counter() - t0) * 1e3
        assert rc == 0, L.lb_last_error()
        total = 0
        p, ln = ctypes.c_void_p(), ctypes.c_size_t()
        for j in range(len(reqs)):
            assert L.lb_exports_get(h, j, ctypes.byref(p), ctypes.byref(ln)) == 0, (j, L.lb_last_error())
            total += ln.value
        L.lb_exports_free(h)
        if step:
            times.append(ms)
    return round(statistics.median(times), 3), total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=40000)
    ap.add_argument("--ops", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--sets", type=int, default=64)
    args = ap.parse_args()
    import loro_b200
    from loro_b200 import api
    from loro_b200.workload import C3Batch
    threads = len(os.sched_getaffinity(0))

    blobs = C3Batch(args.docs, n_ops=args.ops, threads=threads).blobs()
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON, split=1)
    vvs = [batch.oplog_vv(i) for i in range(args.docs)]
    rnd = random.Random(0)
    till = [(i, [(p, 0, rnd.randint(1, c)) for p, c in vv.items()]) for i, vv in enumerate(vvs)]
    till_ms, till_bytes = timed(batch, till, args.steps)

    def two_sided(vv):
        out = []
        for p, c in vv.items():
            a = rnd.randint(0, c - 1)
            out.append((p, a, rnd.randint(a + 1, c)))
        return out
    ranges = [(i, two_sided(vv)) for i, vv in enumerate(vvs)]
    range_ms, range_bytes = timed(batch, ranges, args.steps)
    reexport_ms = batch.timings()["reexport"]
    batch.close()

    one = loro_b200.import_batch([C3Batch(1, n_ops=args.ops, threads=threads).blob(0)],
                                 flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON)
    vv = one.oplog_vv(0)
    sets, seen = [], set()
    while len(sets) < args.sets:
        s = two_sided(vv)
        if tuple(s) not in seen:
            seen.add(tuple(s))
            sets.append((0, s))
    sets_ms, sets_bytes = timed(one, sets, args.steps)
    one.close()

    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power, "docs": args.docs, "ops_per_doc": args.ops, "steps": args.steps,
        "import_reexport_ms": round(reexport_ms, 3),
        "till": {"call_ms": till_ms, "bytes_out": till_bytes},
        "two_sided": {"call_ms": range_ms, "bytes_out": range_bytes},
        "one_doc": {"span_sets": args.sets, "call_ms": sets_ms, "bytes_out": sets_bytes},
    }))


if __name__ == "__main__":
    main()
