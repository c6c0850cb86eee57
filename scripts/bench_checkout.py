#!/usr/bin/env python3
"""Checkout (LoroDoc::checkout(&frontiers) + get_deep_value): device cost of building documents at earlier versions.

Leg 1: `--docs` documents of config C3's shape, each checked out at a random applied id (lb_import_batch_at), against a
plain import of the same batch (lb_import_batch): device milliseconds per phase of both, alternating, `--steps` each
after one warm-up.  Leg 2: ONE C3 document at `--versions` evenly spaced versions in one call (lb_docset_checkout: every
version is a document of its own, one warp each), against the oracle's capped replays of the same versions on the
host's cores.  Prints one JSON line; the card and its power limit are part of it.

  python scripts/bench_checkout.py [--docs 40000] [--ops 10000] [--steps 3] [--versions 1024]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ("h2d", "frame", "decode", "resolve", "classify", "integrate", "tree", "materialise", "total_device")
_doc = None


def _replay(frontiers):
    from tests.checkout_checks import json_at
    return len(json_at(_doc, frontiers))


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                        text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def median_phases(runs):
    return {k: round(statistics.median(r[k] for r in runs), 3) for k in PHASES}


def main():
    global _doc
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=40000)
    ap.add_argument("--ops", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--versions", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import loro_b200
    from loro_b200.workload import C3Batch
    from oracle import OracleDoc
    threads = len(os.sched_getaffinity(0))
    gen = C3Batch(args.docs, n_ops=args.ops, threads=threads)
    blobs = gen.blobs()
    plain = loro_b200.import_batch(blobs)
    rnd = random.Random(0)
    versions = {}
    for i in range(args.docs):
        vv = plain.oplog_vv(i)
        peer = rnd.choice(sorted(vv))
        versions[i] = [(peer, rnd.randrange(vv[peer]))]
    plain.close()
    t_plain, t_at = [], []
    for step in range(args.steps + 1):   # step 0 warms both up
        for leg, out in ((lambda: loro_b200.import_batch(blobs), t_plain),
                         (lambda: loro_b200.import_batch_at(blobs, versions), t_at)):
            b = leg()
            b.fetch_json()
            torch.cuda.synchronize()
            if step:
                out.append(b.timings())
            if step == args.steps and out is t_at:
                bad = sum(1 for i in range(0, args.docs, 97) if b.status(i).code != 0)
                assert bad == 0, f"{bad} sampled documents failed"
            b.close()

    # leg 2: one document at many versions
    blob = C3Batch(1, n_ops=args.ops, threads=threads).blob(0)
    _doc = OracleDoc(1)
    _doc.import_(blob)
    ids = [(p, c) for p, n in sorted(_doc.oplog_vv().items()) for c in range(n)]
    vs = [[ids[(k * len(ids)) // args.versions]] for k in range(args.versions)]
    ds = loro_b200.DocSet()
    ds.import_([blob], [0]).close()
    dev_ms, wall_ms = [], []
    for step in range(args.steps + 1):
        torch.cuda.synchronize()
        t0 = time.time()
        r = ds.checkout([(0, f) for f in vs])
        r.fetch_json()
        torch.cuda.synchronize()
        if step:
            wall_ms.append((time.time() - t0) * 1e3)
            dev_ms.append(r.timings()["total_device"])
        r.close()
    from tests.checkout_checks import _ref_lib
    _ref_lib()
    import multiprocessing as mp
    with mp.get_context("fork").Pool(threads) as pool:
        pool.map(abs, range(threads))
        t0 = time.time()
        pool.map(_replay, vs, chunksize=max(1, len(vs) // (4 * threads)))
        cpu_s = time.time() - t0
    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power,
        "batch": {"docs": args.docs, "ops_per_doc": args.ops, "steps": args.steps,
                  "plain_ms": median_phases(t_plain), "checkout_ms": median_phases(t_at)},
        "one_doc": {"versions": args.versions, "device_ms": round(statistics.median(dev_ms), 3),
                    "wall_ms": round(statistics.median(wall_ms), 3),
                    "oracle_cpu_s": round(cpu_s, 3), "oracle_processes": threads},
    }))


if __name__ == "__main__":
    main()
