#!/usr/bin/env python3
"""export(ExportMode::updates(from)) for many documents: one lb_batch_export_updates call against one
lb_doc_export_updates call per document.

Leg 1: `--docs` documents of config C3's shape, imported with LB_FLAG_EXPORT | LB_FLAG_NO_JSON; every document gets a
seeded random `from` inside its oplog vv, and ONE lb_batch_export_updates call answers all of them (one round): host
wall milliseconds of the call (it ends in a synchronise), median of `--steps` after one warm-up, with the bytes it
returns and the import's `reexport` phase (the all_updates export of every document) beside it.  Leg 2: the same
requests for the first `--sample` documents through lb_doc_export_updates, one call each: milliseconds per call; their
bytes must equal leg 1's.  Leg 3: ONE C3 document at `--versions` distinct versions in one call (one round each).
Prints one JSON line; the card and its power limit are part of it.

  python scripts/bench_export_many.py [--docs 40000] [--ops 10000] [--steps 3] [--sample 256] [--versions 64]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import subprocess
import sys
import time

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


def request_array(reqs):
    """[(doc, {peer: counter}), ...] -> lb_export_request array (+ the span arrays it points into)"""
    from loro_b200 import api
    arr = (api._ExportRequest * max(len(reqs), 1))()
    keep = []
    for j, (doc, frm) in enumerate(reqs):
        spans, k = api._vv_spans(frm)
        keep.append(spans)
        arr[j].doc, arr[j].from_, arr[j].n_from = doc, spans, k
    return arr, keep


def timed_call(batch, arr, n, keep_bytes=False):
    """one lb_batch_export_updates call: (host ms, bytes returned, the blobs when keep_bytes)"""
    L = batch._L
    h = ctypes.c_void_p()
    t0 = time.perf_counter()
    rc = L.lb_batch_export_updates(batch._h, arr, n, ctypes.byref(h))
    ms = (time.perf_counter() - t0) * 1e3
    assert rc == 0, L.lb_last_error()
    total, blobs = 0, []
    p, ln = ctypes.c_void_p(), ctypes.c_size_t()
    for j in range(n):
        assert L.lb_exports_get(h, j, ctypes.byref(p), ctypes.byref(ln)) == 0, (j, L.lb_last_error())
        total += ln.value
        if keep_bytes:
            blobs.append(ctypes.string_at(p.value, ln.value))
    L.lb_exports_free(h)
    return ms, total, blobs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=40000)
    ap.add_argument("--ops", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--versions", type=int, default=64)
    args = ap.parse_args()
    import torch
    import loro_b200
    from loro_b200 import api
    from loro_b200.workload import C3Batch
    threads = len(os.sched_getaffinity(0))

    # leg 1: every document at its own version, one call
    blobs = C3Batch(args.docs, n_ops=args.ops, threads=threads).blobs()
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON, split=1)
    reexport_ms = batch.timings()["reexport"]
    rnd = random.Random(0)
    reqs = [(i, {p: rnd.randint(0, c) for p, c in batch.oplog_vv(i).items()}) for i in range(args.docs)]
    arr, keep = request_array(reqs)
    many_ms = []
    for step in range(args.steps + 1):   # step 0 warms up
        torch.cuda.synchronize()
        ms, out_bytes, many = timed_call(batch, arr, len(reqs), keep_bytes=step == args.steps)
        if step:
            many_ms.append(ms)

    # leg 2: the same requests, one lb_doc_export_updates call each
    sample = reqs[:args.sample]
    for doc, frm in sample[:4]:   # warm-up
        batch.export_updates(doc, frm)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    singles = [batch.export_updates(doc, frm) for doc, frm in sample]
    per_call_ms = (time.perf_counter() - t0) * 1e3 / max(len(sample), 1)
    assert singles == many[:len(sample)], "lb_doc_export_updates differs from lb_batch_export_updates"
    batch.close()

    # leg 3: one document at many versions, one round each
    one = loro_b200.import_batch([C3Batch(1, n_ops=args.ops, threads=threads).blob(0)],
                                 flags=api.LB_FLAG_EXPORT | api.LB_FLAG_NO_JSON)
    vv = one.oplog_vv(0)
    rnd = random.Random(1)
    vs, seen = [], set()
    while len(vs) < args.versions:
        v = {p: rnd.randint(0, c) for p, c in vv.items()}
        key = tuple(sorted(v.items()))
        if key not in seen and any(v.values()):
            seen.add(key)
            vs.append((0, v))
    varr, vkeep = request_array(vs)
    ver_ms = []
    for step in range(args.steps + 1):
        torch.cuda.synchronize()
        ms, ver_bytes, _ = timed_call(one, varr, len(vs))
        if step:
            ver_ms.append(ms)
    one.close()

    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power,
        "many": {"docs": args.docs, "ops_per_doc": args.ops, "steps": args.steps,
                 "call_ms": round(statistics.median(many_ms), 3), "bytes_out": out_bytes,
                 "import_reexport_ms": round(reexport_ms, 3)},
        "single": {"calls": len(sample), "ms_per_call": round(per_call_ms, 3),
                   "equal_to_many": True},
        "one_doc": {"versions": args.versions, "call_ms": round(statistics.median(ver_ms), 3), "bytes_out": ver_bytes},
    }))


if __name__ == "__main__":
    main()
