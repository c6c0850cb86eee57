"""The builds that only large batches select, on the H100 against the oracle, document by document.

Two kernels have a second build that the host picks from the size of the batch:
  * k_seq_integrate<1>: the list integration launches only the CTAs the device holds at once, and their warps take
    documents from a queue, once a batch has more documents than 4 x the resident CTAs (8 per SM);
  * k_exp_encode<1> / k_exp_encode_cut<1>: the re-export encoder under __launch_bounds__(64, 5), once one export pass
    has at least LB_XENC_BOUNDED_MIN_BLOCKS output blocks (k_export.cuh), with its retry encode of the blocks that
    outgrew their staging slot.
Small batches never reach them, so this batch is sized just past both thresholds with small documents, and the
skipped, large and many-peer documents sit among them so that queue warps take them right before healthy ones.  The
oracle's answers are computed here, in worker processes; every call also shows, through torch.profiler, that the
intended build ran, and a small control batch shows the other build's names."""
import gzip
import os
import re

import pytest

from tests import workloads

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TRACE = re.compile(r"\[trace\] export: (\d+) blocks, (\d+) outgrew their staging slot")


def csrc_define(header, name):
    """the value of `#define name <integer>` in loro_b200/csrc/<header>, as the library is built with it"""
    with open(os.path.join(ROOT, "loro_b200", "csrc", header)) as f:
        m = re.search(r"#define\s+%s\s+(\d+)" % name, f.read())
    assert m, f"{name} not found in {header}"
    return int(m.group(1))


def block_count(blob):
    """output blocks of a FastUpdates blob: the length-prefixed blocks after its 22-byte header"""
    n, i = 0, 22
    while i < len(blob):
        ln, sh = 0, 0
        while True:
            c = blob[i]
            i += 1
            ln |= (c & 0x7F) << sh
            sh += 7
            if not c & 0x80:
                break
        i += ln
        n += 1
    return n


def _reference(blob):
    """The oracle's answers for one document (runs in a worker process: touches only the oracle)."""
    import oracle
    from tests.checkout_checks import interesting_ids, json_at
    from tests.range_export_checks import export_in_range
    o = oracle.OracleDoc(1)
    try:
        st = o.import_(blob)
    except oracle.ImportError_ as e:
        return {"code": e.code}
    vv = o.oplog_vv()
    frm = {p: c // 3 for p, c in vv.items()}
    spans = [(p, 0, c - 1) for p, c in vv.items()]   # every peer's last change cut at its end
    ids = interesting_ids(blob)
    at = [ids[len(ids) // 2]] if ids else None
    full = o.export_updates()
    rng = export_in_range(o, spans)
    return {"code": 0, "json": o.json_text(), "vv": vv, "frontiers": sorted(o.frontiers()), "success": st["success"],
            "pending": st["pending"], "export": full, "blocks": block_count(full), "from": frm,
            "export_from": o.export_updates(frm), "spans": spans, "range": rng, "range_blocks": block_count(rng),
            "at": at, "json_at": json_at(o, at) if at else None}


def references(blobs):
    """_reference of every blob, in a pool of spawned processes that ends with this call"""
    import multiprocessing as mp
    from tests import checkout_checks, range_export_checks
    checkout_checks._ref_lib()        # built once here, so that the workers only load them
    range_export_checks._ref_lib()
    with mp.get_context("spawn").Pool(min(os.cpu_count() or 1, 16)) as pool:
        return pool.map(_reference, blobs, chunksize=32)


def kernel_names(fn):
    """fn() under torch.profiler with CUDA activities: (its result, the names of the kernels it launched)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return out, names


def launches(names, kernel, build):
    """launches of template instance kernel<build> among the profiled names, demangled (k<1>(...)) or not (kILi1E)"""
    pat = re.compile(r"(?:\b|\d)%s(?:<%d>|ILi%dE)" % (re.escape(kernel), build, build))
    return sum(1 for n in names if pat.search(n))


def require_builds(names, what, want, other):
    """every kernel of `want` launched, none of `other`; the names seen are printed when not"""
    missing = [k for k in want if not launches(names, *k)]
    unwanted = [k for k in other if launches(names, *k)]
    seen = sorted({n.split("(")[0] for n in names})
    if missing or unwanted:
        print(f"{what}: kernels seen:\n  " + "\n  ".join(seen))
    else:
        print(f"{what}: " + ", ".join(n for n in seen if "k_seq_integrate" in n or "k_exp_encode" in n))
    assert not missing and not unwanted, (what, "missing", missing, "unwanted", unwanted)


def _compare(kind, got, refs, idx, key):
    bad = []
    for i, g in zip(idx, got):
        w = refs[i][key]
        if g != w:
            k = next((j for j in range(min(len(g), len(w))) if g[j] != w[j]), min(len(g), len(w))) \
                if isinstance(g, bytes) else None
            bad.append((i, f"{kind}: differs at byte {k}, lens {len(g) if isinstance(g, bytes) else g} / {len(w)}"))
    assert not bad, (len(bad), bad[:8])


def check_import(batch, refs):
    """status, JSON, vv, frontiers and the all_updates export of every document against the oracle"""
    bad = []
    for i, r in enumerate(refs):
        st = batch.status(i)
        if r["code"]:
            want = {1: 1, 2: 1, 3: 2, 4: 3, 10: (1, 4), 11: 5}[r["code"]]
            if not (st.code == want or (isinstance(want, tuple) and st.code in want)):
                bad.append((i, "code", st.code, r["code"]))
            continue
        if st.code != 0:
            bad.append((i, "code", st.code))
            continue
        if batch.json_bytes(i) != r["json"]:
            bad.append((i, "json"))
        if batch.oplog_vv(i) != r["vv"]:
            bad.append((i, "vv"))
        if batch.oplog_frontiers(i) != r["frontiers"]:
            bad.append((i, "frontiers"))
        if st.success != r["success"] or st.pending != r["pending"]:
            bad.append((i, "status", st, r["success"], r["pending"]))
        if batch.export_updates(i) != r["export"]:
            bad.append((i, "export"))
    assert not bad, (len(bad), bad[:8])


def large_batch(golden_dir):
    """7,500 config C3 documents of 400 ops by 24 peers, and among them, each right before a healthy document: the
    kinds the integration skips (bad checksum, pending only, map only, empty) three times, the automerge trace twice
    (trees deeper than the 12 shared-memory nodes) and four 40-peer histories (peer tables in global memory)"""
    from loro_b200.workload import C3Batch
    g = C3Batch(7500, n_ops=400, n_peers=24, prefix_ops=40, sync_every=20)
    healthy = g.blobs()
    g.close()
    trace = gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read()
    special = workloads.skipped_kinds(healthy[0]) * 3 + [trace, trace]
    special += [workloads.make_doc_history(6300 + k, n_sites=40, n_ops=500, sync_prob=0.04)[0] for k in range(4)]
    special = [special[(7 * k) % len(special)] for k in range(len(special))]   # kinds mixed along the batch
    step = len(healthy) // (len(special) + 1)
    blobs = []
    for k in range(len(special) + 1):
        blobs += healthy[k * step:(k + 1) * step] if k < len(special) else healthy[k * step:]
        if k < len(special):
            blobs.append(special[k])
    assert len(blobs) == len(healthy) + len(special)
    return blobs


SEQ = [("k_seq_integrate", 1)]
SEQ0 = [("k_seq_integrate", 0)]
ENC = [("k_exp_encode", 1)]
ENC0 = [("k_exp_encode", 0)]
CUT = [("k_exp_encode_cut", 1)]
CUT0 = [("k_exp_encode_cut", 0)]


def test_builds_of_large_batches_against_the_oracle(golden_dir, monkeypatch, capfd):
    import time
    import torch
    import loro_b200
    from loro_b200 import api
    t0 = time.time()
    torch.cuda.init()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    threshold = csrc_define("k_export.cuh", "LB_XENC_BOUNDED_MIN_BLOCKS")
    seq_minb = csrc_define("k_seq.cuh", "LB_SEQ_MINB")   # CTAs of k_seq_integrate resident per SM at most
    blobs = large_batch(golden_dir)
    assert len(blobs) > 4 * seq_minb * sms, (len(blobs), sms)   # more documents than the resident warps: the queue
    refs = references(blobs)
    ok = [i for i, r in enumerate(refs) if r["code"] == 0]
    assert sum(refs[i]["blocks"] for i in ok) >= threshold
    assert sum(refs[i]["range_blocks"] for i in ok) >= threshold
    print(f"{len(blobs)} documents, {sms} SMs; oracle: {sum(refs[i]['blocks'] for i in ok)} blocks in export, "
          f"{sum(refs[i]['range_blocks'] for i in ok)} in range export; references {time.time() - t0:.1f} s")

    # (a) the import with its all_updates export
    batch, names = kernel_names(lambda: loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, split=1))
    require_builds(names, "import", SEQ + ENC, SEQ0 + ENC0)
    check_import(batch, refs)
    # (b) exports from {peer: counter // 3}
    _compare("export from", batch.export_updates_many([(i, refs[i]["from"]) for i in ok]), refs, ok, "export_from")
    # (c) range exports whose spans end inside the last change of every peer
    got, names = kernel_names(lambda: batch.export_updates_in_range_many([(i, refs[i]["spans"]) for i in ok]))
    require_builds(names, "range export", CUT, CUT0 + ENC0)
    _compare("range export", got, refs, ok, "range")
    exported = [batch.export_updates(i) for i in ok]
    batch.close()

    # (d) the same import with the staging slots capped at 1,000 bytes: some blocks of the bounded build go through the
    # retry encode
    monkeypatch.setenv("LB_EXPORT_STAGE_CAP", "1000")
    monkeypatch.setenv("LB_PHASE_TRACE", "1")
    earlier = capfd.readouterr().out
    again, names = kernel_names(lambda: loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, split=1))
    m = TRACE.findall(capfd.readouterr().err)
    print(earlier, end="")   # this test's lines so far, read together with what came before the trace
    monkeypatch.delenv("LB_EXPORT_STAGE_CAP")
    monkeypatch.delenv("LB_PHASE_TRACE")
    assert len(m) == 1, m
    n_blocks, n_ovf = int(m[0][0]), int(m[0][1])
    assert n_blocks >= threshold and 0 < n_ovf < n_blocks, (n_blocks, n_ovf)
    require_builds(names, "import with capped slots", SEQ + ENC, SEQ0 + ENC0)
    assert launches(names, "k_exp_encode", 1) == 2, "the encode and its retry, both in the bounded build"
    _compare("export with capped slots", [again.export_updates(i) for i in ok], refs, ok, "export")
    assert [again.export_updates(i) for i in ok] == exported
    again.close()

    # (e) checkout at one mid-history id of every document that has one
    req = {i: refs[i]["at"] for i in ok if refs[i]["at"]}
    at, names = kernel_names(lambda: loro_b200.import_batch_at(blobs, req))
    require_builds(names, "checkout", SEQ, SEQ0)
    bad = []
    for i in ok:
        st = at.status(i)
        if i not in req:
            if st.code != 0 or at.json_bytes(i) != refs[i]["json"]:
                bad.append((i, "latest", st.code))
        elif refs[i]["json_at"] is None:
            if st.code != 7:     # FrontiersNotFound, as the oracle
                bad.append((i, "not found", st.code))
        elif st.code != 0 or at.json_bytes(i) != refs[i]["json_at"]:
            bad.append((i, "at", req[i], st.code))
        elif at.oplog_vv(i) != refs[i]["vv"]:
            bad.append((i, "vv"))
    at.close()
    assert not bad, (len(bad), bad[:8])
    print(f"large batch: {time.time() - t0:.1f} s")


def test_control_batch_takes_the_small_builds():
    """64 documents of the same shape: the one-warp-per-document integration and the unbounded encoders, so that the
    names matched above are the ones the profiler reports for these kernels"""
    import loro_b200
    from loro_b200 import api
    from loro_b200.workload import C3Batch
    g = C3Batch(64, n_ops=400, n_peers=24, prefix_ops=40, sync_every=20)
    blobs = g.blobs()
    g.close()
    refs = [_reference(b) for b in blobs]
    ok = list(range(len(blobs)))
    batch, names = kernel_names(lambda: loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, split=1))
    require_builds(names, "control import", SEQ0 + ENC0, SEQ + ENC)
    check_import(batch, refs)
    got, names = kernel_names(lambda: batch.export_updates_in_range_many([(i, refs[i]["spans"]) for i in ok]))
    require_builds(names, "control range export", CUT0, CUT + ENC)
    _compare("range export", got, refs, ok, "range")
    batch.close()
