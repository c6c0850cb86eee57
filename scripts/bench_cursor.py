#!/usr/bin/env python3
"""Cursors (lb_batch_cursor_pos): what LB_FLAG_CURSORS costs at import, and how fast a query call answers.

1. A C3 batch (`--docs` documents) is imported without and with LB_FLAG_CURSORS, alternating, `--steps` times each after
   one warm-up of both: median device milliseconds of the whole import (total_device) and of the import-time cursor
   phase (lb_timings.cursors).
2. On the flagged batch, one call answers `--cursors` cursors spread over every document (ids drawn from each
   document's oplog, so visible, deleted and foreign ones): median host wall time of the call over `--steps` calls
   (upload, kernel, download), and the device time of k_cursor_query from torch.profiler in a separate call.
3. The reference restated on the host (tests/cursor_ref.cpp, a process per core) answers the same cursors for the
   first `--ref-docs` documents, each document imported and replayed first, as a server without this engine would.
Prints one JSON line; the card, its power limit and its SM clock are part of it.

  python scripts/bench_cursor.py [--docs 40000] [--cursors 1000000] [--steps 3] [--ref-docs 256]
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

_work = None


def _ref(i):
    from tests.checkout_checks import oracle_doc
    from tests.cursor_checks import cursor_pos_ref
    blob, cs = _work[i]
    return len(cursor_pos_ref(oracle_doc([blob]), cs))


def clocks():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader",
                                        "-i", "0"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=40000)
    ap.add_argument("--cursors", type=int, default=1000000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--ref-docs", type=int, default=256)
    args = ap.parse_args()
    global _work
    import torch
    import loro_b200
    from loro_b200.api import LB_FLAG_ATTRIBUTION, LB_FLAG_CURSORS
    from loro_b200.workload import C3Batch
    from scripts.bench_checkout import card
    from tests.cursor_checks import sample_cursors
    threads = len(os.sched_getaffinity(0))
    blobs = C3Batch(args.docs, n_ops=10000, threads=threads).blobs()
    # ---- 1. import cost
    plain, cur = [], []
    b = None
    for step in range(args.steps + 1):   # step 0 warms both up
        for flags, out in ((0, plain), (LB_FLAG_CURSORS, cur)):
            if b is not None:
                b.close()
            b = loro_b200.import_batch(blobs, flags=flags, split=1)
            b.fetch_json()
            torch.cuda.synchronize()
            if step:
                out.append(b.timings())
    # ---- 2. one call for all cursors (b is the last flagged batch)
    one = loro_b200.import_batch(blobs[:1], flags=LB_FLAG_ATTRIBUTION)
    cids = [c for c in one.attribution(0) if c.endswith((":Text", ":List"))]
    one.close()
    rnd = random.Random(41)
    per_doc = max(1, args.cursors // len(blobs))
    reqs, mine = [], {}
    for i in range(len(blobs)):
        cs = sample_cursors(rnd, cids, b.oplog_vv(i), per_doc)
        if i < args.ref_docs:
            mine[i] = cs
        reqs += [(i,) + c for c in cs]
    b.cursor_pos(reqs[:1000])   # warm-up
    walls = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        got = b.cursor_pos(reqs)
        walls.append((time.perf_counter() - t0) * 1e3)
    # the binding's own time (building and reading the ctypes arrays) is not the engine's: the C call alone
    import ctypes
    from loro_b200 import api
    from loro_b200.api import parse_container_id
    n = len(reqs)
    arr = (api._Cursor * n)()
    names = {}
    for k, (doc, cid, tid, side) in enumerate(reqs):
        is_root, name, peer, counter, ctype = parse_container_id(cid)
        c = arr[k]
        c.doc, c.is_root, c.type, c.side = doc, is_root, ctype, side
        if is_root:
            names.setdefault(name, name)
            c.name, c.name_len = names[name], len(name)
        else:
            c.peer, c.counter = peer, counter
        if tid is not None:
            c.has_id, c.id_peer, c.id_counter = 1, tid[0], tid[1]
    res = (api._CursorResult * n)()
    c_walls = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        assert b._L.lb_batch_cursor_pos(b._h, arr, n, res) == 0
        c_walls.append((time.perf_counter() - t0) * 1e3)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        b._L.lb_batch_cursor_pos(b._h, arr, n, res)
        torch.cuda.synchronize()
    kern_us = sum(e.device_time_total for e in prof.key_averages() if "k_cursor_query" in e.key)
    n_deleted = sum(u is not None for _, _, _, u in got)
    b.close()
    # ---- 3. the reference on the host's cores
    _work = [(blobs[i], mine[i]) for i in sorted(mine)]
    from tests.cursor_checks import _ref_lib
    _ref_lib()
    import multiprocessing as mp
    with mp.get_context("fork").Pool(threads) as pool:
        pool.map(abs, range(threads))
        t0 = time.time()
        pool.map(_ref, range(len(_work)), chunksize=max(1, len(_work) // (4 * threads)))
        cpu_s = time.time() - t0
    ref_cursors = sum(len(cs) for _, cs in _work)

    def med(runs, k):
        return round(statistics.median(r[k] for r in runs), 3)
    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power, "sm_clock_now_max": clocks(), "config": "C3", "docs": len(blobs),
        "steps": args.steps,
        "plain_total_device_ms": med(plain, "total_device"), "cursors_total_device_ms": med(cur, "total_device"),
        "cursors_phase_ms": med(cur, "cursors"), "cursors_phase_ms_runs": [round(r["cursors"], 3) for r in cur],
        "plain_total_device_ms_runs": [round(r["total_device"], 3) for r in plain],
        "cursors_total_device_ms_runs": [round(r["total_device"], 3) for r in cur],
        "query_cursors": n, "query_deleted_targets": n_deleted,
        "query_python_call_ms": round(statistics.median(walls), 3), "query_c_call_ms": round(statistics.median(c_walls), 3),
        "query_kernel_ms": round(kern_us / 1e3, 3),
        "query_cursors_per_s": round(n / (statistics.median(c_walls) / 1e3)),
        "reference_docs": len(_work), "reference_cursors": ref_cursors, "reference_cpu_s": round(cpu_s, 3),
        "reference_processes": threads, "reference_cursors_per_s": round(ref_cursors / cpu_s, 1) if cpu_s else None,
    }))


if __name__ == "__main__":
    main()
