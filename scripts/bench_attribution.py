#!/usr/bin/env python3
"""Attribution (lb_doc_attribution): device cost of the attribution phase against the whole import.

For config C3 (`--docs` documents) and config C5 (`--c5-docs` documents), the same batch is imported without and with
LB_FLAG_ATTRIBUTION, alternating, `--steps` times each after one warm-up of both; reported are the median device
milliseconds of the attribution phase and of the whole import (total_device), the attribution bytes per document, and
the reference's host throughput (tests/attribution_ref.cpp on all the host's cores) on a sample of the same documents.
Prints one JSON line; the card and its power limit are part of it.

  python scripts/bench_attribution.py [--docs 40000] [--c5-docs 10000] [--steps 3] [--ref-docs 512]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_blobs = None


def _ref(i):
    from tests.attribution_checks import attribution_at
    from tests.checkout_checks import oracle_doc
    return len(attribution_at(oracle_doc([_blobs[i]])))


def leg(name, blobs, steps, ref_docs, threads):
    global _blobs
    import torch
    import loro_b200
    from loro_b200.api import LB_FLAG_ATTRIBUTION
    plain, attr = [], []
    attr_bytes = 0
    for step in range(steps + 1):   # step 0 warms both up
        for flags, out in ((0, plain), (LB_FLAG_ATTRIBUTION, attr)):
            b = loro_b200.import_batch(blobs, flags=flags, split=1)
            b.fetch_json()
            if flags:
                attr_bytes = sum(len(b.attribution_bytes(i)) for i in range(b.n_docs))
            torch.cuda.synchronize()
            if step:
                out.append(b.timings())
            b.close()
    # the reference on the host's cores, on the first ref_docs documents
    _blobs = blobs[:ref_docs]
    from tests.attribution_checks import _ref_lib
    _ref_lib()
    import multiprocessing as mp
    with mp.get_context("fork").Pool(threads) as pool:
        pool.map(abs, range(threads))
        t0 = time.time()
        pool.map(_ref, range(len(_blobs)), chunksize=max(1, len(_blobs) // (4 * threads)))
        cpu_s = time.time() - t0

    def med(runs, k):
        return round(statistics.median(r[k] for r in runs), 3)
    return {
        "config": name, "docs": len(blobs), "steps": steps,
        "plain_total_device_ms": med(plain, "total_device"), "plain_materialise_ms": med(plain, "materialise"),
        "attr_total_device_ms": med(attr, "total_device"), "attr_materialise_ms": med(attr, "materialise"),
        "attribution_ms": med(attr, "attribution"),
        "attribution_ms_runs": [round(r["attribution"], 3) for r in attr],
        "attribution_bytes_per_doc": round(attr_bytes / max(1, len(blobs)), 1),
        "reference_docs": len(_blobs), "reference_cpu_s": round(cpu_s, 3), "reference_processes": threads,
        "reference_docs_per_s": round(len(_blobs) / cpu_s, 1) if cpu_s else None,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=40000)
    ap.add_argument("--c5-docs", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--ref-docs", type=int, default=512)
    args = ap.parse_args()
    from loro_b200.workload import C3Batch, C5Batch
    from scripts.bench_checkout import card
    threads = len(os.sched_getaffinity(0))
    legs = [leg("C3", C3Batch(args.docs, n_ops=10000, threads=threads).blobs(), args.steps, args.ref_docs, threads)]
    legs.append(leg("C5", C5Batch(args.c5_docs, threads=threads).blobs(), args.steps, args.ref_docs, threads))
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "legs": legs}))


if __name__ == "__main__":
    main()
