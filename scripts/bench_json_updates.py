#!/usr/bin/env python3
"""LoroDoc::export_json_updates on the device (lb_batch_export_json_updates) against the reference's JSON export on
the CPU.

Leg 1: `--docs` documents of config C3's shape, imported with LB_FLAG_EXPORT | LB_FLAG_NO_JSON; ONE call exports all
updates of every document (start = the empty version, end = the oplog vv): host wall milliseconds of the call (it ends
in a synchronise), median of `--steps` after one warm-up, and the JSON bytes it returns.  Leg 2: ONE C3 document at
`--ranges` seeded random version ranges in one call, timed the same way.  Leg 3: the reference's JSON export
(tests/json_updates_ref.cpp on the oracle, the C++ restatement of the reference; there is no Rust toolchain here) of the
first `--sample` documents of leg 1, one process per host core: documents per second, and its text must equal the
engine's.  `--lib` times another build of the library.  Prints one JSON line; the card and its power limit are part of
it.

  python scripts/bench_json_updates.py [--docs 4096] [--ops 10000] [--steps 3] [--ranges 64] [--sample 64] [--lib PATH]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                        text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def timed(batch, reqs, steps):
    """median host ms of one export_json_updates_many call over `steps` calls after one warm-up, and the last texts"""
    import torch
    times, out = [], None
    for step in range(steps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = batch.export_json_updates_many(reqs)
        ms = (time.perf_counter() - t0) * 1e3
        if step:
            times.append(ms)
    assert all(isinstance(o, str) for o in out), [o for o in out if not isinstance(o, str)][:1]
    return statistics.median(times), out


def _reference(blob):
    from tests import json_updates_checks as jc
    return jc.export_json_updates(jc.oracle_doc([blob]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=4096)
    ap.add_argument("--ops", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--ranges", type=int, default=64)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--lib", default=None)
    args = ap.parse_args()
    import loro_b200
    from loro_b200 import api
    from loro_b200.workload import C3Batch
    from tests import json_updates_checks as jc
    threads = len(os.sched_getaffinity(0))

    blobs = C3Batch(args.docs, n_ops=args.ops, threads=threads).blobs()
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON, split=1, lib_path=args.lib)
    many_ms, texts = timed(batch, [(i, None, None) for i in range(args.docs)], args.steps)
    many_bytes = sum(len(t.encode()) for t in texts)

    vv = batch.oplog_vv(0)
    rng = random.Random(1)
    ranges = [(0,) + jc.random_range(rng, vv) for _ in range(args.ranges)]
    range_ms, range_texts = timed(batch, ranges, args.steps)
    range_bytes = sum(len(t.encode()) for t in range_texts)

    sample = blobs[:args.sample]
    with ProcessPoolExecutor(threads) as ex:
        list(ex.map(_reference, sample[:threads]))   # warm-up: the reference library is built and loaded per process
        t0 = time.perf_counter()
        ref = list(ex.map(_reference, sample))
        ref_s = time.perf_counter() - t0
    assert ref == texts[:len(sample)], "engine text differs from the reference"

    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power,
        "all_updates": {"docs": args.docs, "ops_per_doc": args.ops, "steps": args.steps,
                        "call_ms": round(many_ms, 3), "json_bytes": many_bytes},
        "one_doc_ranges": {"ranges": args.ranges, "call_ms": round(range_ms, 3), "json_bytes": range_bytes},
        "reference_cpu": {"docs": len(sample), "processes": threads, "seconds": round(ref_s, 3),
                          "docs_per_s": round(len(sample) / ref_s, 1), "equal_to_engine": True},
    }))


if __name__ == "__main__":
    main()
