#!/usr/bin/env python3
"""Phase 6 (materialise) launch by launch: one step of a bench.py config under torch.profiler (CUDA activities).

The batch is laid out in HBM as bench.py lays it out, one step warms up, and the next step is traced.  Reported per
launch of the phase: `k_json` pass 0 (count), `k_json_padlen`, the scan of the padded lengths, `k_json` pass 1
(write) and `k_doc_hash`; the gap between the end of the scan and the start of the write pass (the download of the
JSON total and the allocation of the JSON buffer); the phase's span on the device; and the JSON bytes of the step.
Prints one JSON line; the card and its power limit are part of it.  `--trace DIR` also writes the Chrome trace there.

  python scripts/profile_materialise.py --config C3 [--docs N] [--trace DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def phase6(kernels):
    """The phase's launches from the step's kernels in start order: the last k_json pair and what lies between."""
    idx = [i for i, k in enumerate(kernels) if k["name"].startswith("k_json(") or k["name"] == "k_json"]
    if len(idx) < 2:
        raise SystemExit(f"expected two k_json launches in the step, found {len(idx)}")
    i0, i1 = idx[-2], idx[-1]
    between = kernels[i0 + 1:i1]
    after = [k for k in kernels[i1 + 1:] if k["name"].startswith("k_doc_hash")][:1]
    if not after:
        raise SystemExit("no k_doc_hash launch after the write pass")
    return kernels[i0], between, kernels[i1], after[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C2", "C3", "C5"])
    ap.add_argument("--docs", type=int, default=0)
    ap.add_argument("--trace", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import loro_b200
    sys.argv = [sys.argv[0], "--config", a.config, "--docs", str(a.docs)]
    args = bench.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    n_docs = bench.default_docs(args, 1)
    gen, distinct, _ = bench.make_workload(args, 0, 1, n_docs)
    idx = np.arange(n_docs) % distinct
    lens = gen.lens[idx].astype(np.uint32)
    src = torch.from_numpy(np.ascontiguousarray(gen.bytes)).to(dev)
    span = (int(src.numel()) + 15) & ~15
    reps = (n_docs + distinct - 1) // distinct
    d_bytes = torch.zeros(span * reps + 64, dtype=torch.uint8, device=dev)
    for c in range(reps):
        d_bytes[c * span:c * span + src.numel()] = src
    offs = (gen.offsets.astype(np.uint64)[idx] + (np.arange(n_docs) // distinct).astype(np.uint64) * np.uint64(span))
    del src
    xflags = loro_b200.api.LB_FLAG_EXPORT

    def step():
        b = loro_b200.import_batch_device(d_bytes.data_ptr(), offs, lens, device=0, flags=xflags, keep=d_bytes)
        c = b.counters()
        assert c["docs_ok"] == n_docs, c
        tm = b.timings()
        b.close()
        return tm, c["json_bytes"]

    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tm, json_total = step()
        torch.cuda.synchronize()
    if a.trace:
        os.makedirs(a.trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(a.trace, f"materialise_{a.config}.pt.trace.json"))
    kernels = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.name.startswith("k_"):
            kernels.append({"name": e.name, "t0": e.time_range.start, "t1": e.time_range.end})
    kernels.sort(key=lambda k: k["t0"])
    count, between, write, dhash = phase6(kernels)

    def ms(k):
        return round((k["t1"] - k["t0"]) / 1e3, 3)
    line = {
        "config": a.config, "docs": n_docs, "card": card(),
        "k_json_count_ms": ms(count),
        "between": [{"name": k["name"].split("(")[0], "ms": ms(k)} for k in between],
        "gap_before_write_ms": round((write["t0"] - (between[-1]["t1"] if between else count["t1"])) / 1e3, 3),
        "k_json_write_ms": ms(write),
        "k_doc_hash_ms": ms(dhash),
        "phase_span_ms": round((dhash["t1"] - count["t0"]) / 1e3, 3),
        "materialise_event_ms": round(tm["materialise"], 3),
        "json_bytes": json_total,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
