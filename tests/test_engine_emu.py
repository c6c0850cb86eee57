"""Functional tests of the product's kernels compiled against the SIMT emulator (tests/emu): logic parity
with the oracle in the GPU-less container.  The same checks run on the real CUDA build in test_engine_gpu.py.
The emulated library is test infrastructure only -- loro_b200 never loads it by default."""
import os
import subprocess
import sys

import pytest

import oracle
from oracle import OracleDoc
from tests import workloads
from tests.engine_checks import check_batch_against_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def test_small_mixed_doc():
    a = OracleDoc(1)
    t = a.get_text("text"); a.text_insert(t, 0, "Hello"); a.text_insert(t, 5, " World")
    l = a.get_list("list"); a.list_insert(l, 0, 1, 2, 3); a.delete(l, 1, 1)
    m = a.get_map("map"); a.map_set(m, "k", 5); a.map_set(m, "z", "str"); a.map_delete(m, "k")
    b = check_batch_against_oracle([a.export_updates()], lib_path=EMU)
    assert b.get_deep_value(0) == {"text": "Hello World", "list": [1, 3], "map": {"z": "str"}}
    c = b.counters()
    assert c["atom_ops"] == a.len_ops() and c["docs_ok"] == 1


def test_fugue_known_answers():
    """crates/loro-internal/tests/fugue.rs through the engine."""
    a, b = OracleDoc(0), OracleDoc(1)
    for ch in "olleH":
        a.text_insert(a.get_text("text"), 0, ch)
    for ch in "!dlroW ":
        b.text_insert(b.get_text("text"), 0, ch)
    workloads.merge(a, b)
    a2, b2, c2 = OracleDoc(0), OracleDoc(1), OracleDoc(2)
    c2.text_insert(c2.get_text("text"), 0, "2")
    workloads.merge(a2, c2)
    a2.text_insert(a2.get_text("text"), 0, "1")
    b2.text_insert(b2.get_text("text"), 0, "b")
    workloads.merge(a2, b2)
    batch = check_batch_against_oracle([a.export_updates(), a2.export_updates()], lib_path=EMU)
    assert batch.get_deep_value(0) == {"text": "Hello World!"}
    assert batch.get_deep_value(1) == {"text": "b12"}


def test_pending_and_bad_blobs():
    a = OracleDoc(1)
    a.text_insert(a.get_text("t"), 0, "abc")
    a.commit()
    vv1 = a.oplog_vv()
    a.text_insert(a.get_text("t"), 3, "def")
    full, tail = a.export_updates(), a.export_updates(vv1)
    bad_sum = full[:30] + bytes([full[30] ^ 1]) + full[31:]
    batch = check_batch_against_oracle([full, tail, bad_sum, b"lor0" + full[4:], full[:10], b""], lib_path=EMU)
    assert batch.status(1).pending == {1: (3, 6)} and batch.status(1).success == {}
    assert batch.get_deep_value(1) == {"t": ""}  # root registered at decode time, nothing applied
    assert [batch.status(i).code for i in range(2, 6)] == [2, 1, 1, 1]


@pytest.mark.parametrize("seed", range(6))
def test_random_multi_site_histories(seed):
    blobs, jsons = [], []
    for k in range(4):
        blob, js, vv, _ = workloads.make_doc_history(seed * 100 + k, n_sites=2 + (seed + k) % 3, n_ops=120 + 40 * k)
        blobs.append(blob)
        jsons.append(js)
    check_batch_against_oracle(blobs, lib_path=EMU, expect_json=jsons)


def test_c1_two_peer_list_sync_small():
    blob, js = workloads.c1_two_peer_list(seed=1, n_each=150)
    check_batch_against_oracle([blob], lib_path=EMU, expect_json=[js])


def test_device_entry_point_layout():
    import loro_b200
    blobs = [workloads.make_doc_history(9000 + k, n_sites=3, n_ops=80)[0] for k in range(5)]
    host = loro_b200.import_batch(blobs, lib_path=EMU)
    buf, offs, lens = loro_b200.pack_blobs(blobs)
    dev = loro_b200.import_batch_device(buf.ctypes.data, offs, lens, lib_path=EMU, keep=buf)
    for i in range(len(blobs)):
        assert dev.status(i) == host.status(i)
        assert dev.json_bytes(i) == host.json_bytes(i)
    assert dev.counters()["state_hash"] == host.counters()["state_hash"]


def test_longer_concurrent_branches():
    blob, js, _, _ = workloads.make_doc_history(7001, n_sites=3, n_ops=900, sync_prob=0.006)
    check_batch_against_oracle([blob], lib_path=EMU, expect_json=[js])


def test_more_than_32_peers():
    """40 concurrent sites: peers beyond the 32 whose atom bases / tracker versions are cached in shared memory
    take the global-memory paths of the integration kernel (C4 shape at test size)."""
    from tests.export_checks import check_export_against_oracle
    blobs, js = [], []
    for i in range(3):
        blob, j, _, _ = workloads.make_doc_history(4200 + i, n_sites=40, n_ops=900, sync_prob=0.04)
        blobs.append(blob)
        js.append(j)
    check_batch_against_oracle(blobs, expect_json=js, lib_path=EMU)
    check_export_against_oracle(blobs, lib_path=EMU)


def test_automerge_trace_end_content(golden_dir):
    """C2 shape on one document (259,778 patches): exercises multi-level trees and node spill past the
    shared-memory cache."""
    import gzip, json
    import loro_b200
    blob = gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read()
    end = json.load(gzip.open(os.path.join(golden_dir, "automerge_trace.json.gz")))["endContent"]
    b = loro_b200.import_batch([blob], lib_path=EMU)
    assert b.status(0).code == 0 and b.get_deep_value(0) == {"text": end}
    assert b.counters()["atom_ops"] == 259778


def test_generator_three_way_agreement():
    """The workload generator's origin-based Fugue replicas, the oracle's eg-walker replay and the engine's
    kernels must agree on the final state of C3 documents (three independent formulations)."""
    import loro_b200
    from loro_b200.workload import C3Batch
    gen = C3Batch(6, n_ops=1200, want_json=True, threads=4)
    blobs = gen.blobs()
    batch = check_batch_against_oracle(blobs, lib_path=EMU)
    for i in range(gen.n_docs):
        assert batch.json_bytes(i) == gen.expected_json(i)
    assert batch.counters()["atom_ops"] == gen.atom_ops


def test_host_staging_ring_small_slots():
    """host_stage.hpp: multi-slot / multi-thread gather + scatter (LB_STAGE_SLOT shrinks the pinned slots) gives the
    same bytes as the single-slot path."""
    import hashlib, sys
    blobs = [workloads.make_doc_history(900 + i, n_sites=2, n_ops=80)[0] for i in range(6)]
    import loro_b200
    b = loro_b200.import_batch(blobs, lib_path=EMU)
    want = hashlib.sha256(b"\n".join(b.json_bytes(i) for i in range(len(blobs)))).hexdigest()
    code = (
        "import sys, hashlib, pickle; sys.path.insert(0, %r); import loro_b200\n"
        "blobs = pickle.load(open(sys.argv[1], 'rb'))\n"
        "b = loro_b200.import_batch(blobs, lib_path=%r)\n"
        "print(hashlib.sha256(b'\\n'.join(b.json_bytes(i) for i in range(len(blobs)))).hexdigest())\n"
    ) % (os.path.dirname(HERE), EMU)
    import pickle, tempfile
    with tempfile.NamedTemporaryFile(suffix=".pkl") as f:
        pickle.dump(blobs, f); f.flush()
        for slot in ("64", "4096"):
            out = subprocess.check_output([sys.executable, "-c", code, f.name], env=dict(os.environ, LB_STAGE_SLOT=slot))
            assert out.decode().strip() == want, slot


def _per_peer_blobs(seed, n_sites=3, n_ops=300):
    """One history, exported as one blob per peer (each holds only that peer's changes, which depend on the
    others'): the import_batch shape of SURVEY 8d's C3 variant."""
    blob, js, vv, sites = workloads.make_doc_history(seed, n_sites=n_sites, n_ops=n_ops)
    full = sites[0]
    tot = full.oplog_vv()
    parts = [full.export_updates({q: c for q, c in tot.items() if q != p}) for p in tot]
    return blob, js, tot, parts


def test_import_batch_groups_blobs_by_doc_id():
    """LoroDoc::import_batch: several update blobs into one document, in any order, with a duplicate; changes whose
    dependencies sit in a later blob resolve inside the batch (pending_changes.rs)."""
    import random
    import loro_b200
    blobs, ids, want = [], [], []
    for d in range(5):
        whole, js, tot, parts = _per_peer_blobs(3100 + d, n_sites=2 + d % 3, n_ops=150 + 40 * d)
        random.Random(d).shuffle(parts)
        if d % 2:
            parts.append(parts[0])          # the same update twice: a no-op (issue.rs:257-264)
        for p in parts:
            blobs.append(p)
            ids.append(1000 + d)
        want.append((js, tot))
    # interleave documents: grouping is by id, not by position
    order = list(range(len(blobs)))
    random.Random(99).shuffle(order)
    b = loro_b200.import_batch([blobs[i] for i in order], doc_ids=[ids[i] for i in order], lib_path=EMU)
    assert b.n_docs == 5
    first_seen = []
    for i in order:
        if ids[i] not in first_seen:
            first_seen.append(ids[i])
    saw_pending = 0
    for k, did in enumerate(first_seen):
        js, tot = want[did - 1000]
        ost = OracleDoc(77).import_batch([blobs[i] for i in order if ids[i] == did])   # same arrival order as the engine's
        st = b.status(k)
        # the status folds the per-blob statuses the way LoroDoc::import_batch does: a change parked by one blob and
        # released by a later one still shows up in `pending` (encoding.rs:252-257, loro.rs:1228-1258)
        assert st.code == 0 and st.success == ost["success"] and st.pending == ost["pending"], (did, st, ost)
        saw_pending += ost["pending"] is not None
        assert b.json_bytes(k) == js
        assert b.oplog_vv(k) == tot
    assert saw_pending > 0
    # a missing part leaves the dependants pending, exactly as a lone import would
    whole, js, tot, parts = _per_peer_blobs(3200, n_sites=3, n_ops=200)
    b2 = loro_b200.import_batch(parts[:2], doc_ids=[7, 7], lib_path=EMU)
    ref = OracleDoc(5)
    ost = ref.import_batch(parts[:2])
    assert b2.n_docs == 1 and b2.json_bytes(0) == ref.json_text()
    assert b2.oplog_vv(0) == ref.oplog_vv()
    assert b2.status(0).success == ost["success"] and b2.status(0).pending == ost["pending"], (b2.status(0), ost)


def test_import_batch_full_blob_plus_overlapping_sliced_blob():
    """A full history next to `export(updates(vv))` of the same history: the sliced copy A[3..n) of a merged change
    is a duplicate that must be dropped, and a dependency on an atom it covers resolves to the applied original
    (round-1 advisor finding: lamport_of picked the dropped record)."""
    import loro_b200
    a, b = OracleDoc(1), OracleDoc(2)
    t = a.get_text("t")
    a.text_insert(t, 0, "0123456789")
    a.commit()
    workloads.merge(b, a)
    tb = b.get_text("t")
    b.text_insert(tb, 5, "xyz")      # depends on 1@9 through the frontier
    b.commit()
    workloads.merge(a, b)
    a.text_insert(t, 2, "Q")
    a.commit()
    full = a.export_updates()
    sliced = a.export_updates({1: 3})
    for blobs in ([full, sliced], [sliced, full]):
        ref = OracleDoc(9)
        ost = ref.import_batch(blobs)
        r = loro_b200.import_batch(blobs, doc_ids=[5, 5], lib_path=EMU)
        assert r.n_docs == 1 and r.status(0).code == 0
        assert r.status(0).success == ost["success"] and r.status(0).pending == ost["pending"], (r.status(0), ost)
        assert r.json_bytes(0) == ref.json_text()
        assert r.oplog_vv(0) == ref.oplog_vv()


def test_rows_straddling_change_boundary_are_corrupt():
    """A checksummed block whose change lengths disagree with its op rows (advisor finding: an out-of-bounds atom
    write of attacker-chosen size) must fail the document, not the batch."""
    import struct
    import loro_b200
    from loro_b200 import api
    a = OracleDoc(1)
    t = a.get_text("t")
    a.text_insert(t, 0, "x" * 800)
    a.commit()
    b = OracleDoc(2)
    b.text_insert(b.get_text("t"), 0, "y")
    b.commit()
    workloads.merge(a, b)
    a.text_insert(t, 3, "abcde")     # second change of peer 1 in the same block (has a foreign dep -> no merge)
    a.commit()
    blob = bytearray(a.export_updates())
    # find the `a0 06` (= 800) change-length varint of the header and patch it to 1, then re-seal
    i = blob.find(bytes([0xA0, 0x06]), 22)
    assert i > 0
    patched = blob[:i] + bytes([0x01]) + blob[i + 2:]
    # the block and section length prefixes shrink by one byte: rebuild them by re-framing through the oracle's dump
    # is overkill -- instead patch in place keeping the length (0x81 0x00 is a non-canonical varint for 1)
    patched = blob[:i] + bytes([0x81, 0x00]) + blob[i + 2:]
    h = oracle.i64s(oracle.codec("xxh32", bytes(patched[20:]), 0x4F524F4C))[0] & 0xFFFFFFFF
    patched = bytes(patched[:16]) + struct.pack("<I", h) + bytes(patched[20:])
    good = a.export_updates()
    r = loro_b200.import_batch([patched, good], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    assert r.status(0).code in (1, 4), r.status(0)
    assert r.status(1).code == 0


def test_config_c4_shape_many_fully_concurrent_branches():
    """BASELINE config C4 in small: one Text document, a pasted base and 40 peers (more than a warp has lanes) that
    edit their own copy of it without ever syncing -- one merge of 40 fully concurrent branches; state and re-exported
    bytes equal the oracle's, and the generator's own encoder agrees with the oracle's export byte for byte."""
    from loro_b200.workload import C4Doc
    from tests.export_checks import check_export_against_oracle
    g = C4Doc(base_chars=6000, n_peers=40, edits=120)
    blob = g.blob(0)
    o = OracleDoc(1)
    o.import_(blob)
    assert not o.inconsistent_delete() and o.export_updates() == blob
    b = check_batch_against_oracle([blob], lib_path=EMU)
    assert b.counters()["atom_ops"] == g.atom_ops
    check_export_against_oracle([blob], lib_path=EMU)


def test_decode_tables_against_the_oracle_decoder():
    """Decode SoA, table by table (lb_debug_table): every row / change / dependency column the decode kernels write
    equals what the oracle's block decoder reads from the same blobs -- a decode fault is localised here, not only
    through the state JSON and the re-exported bytes downstream."""
    import numpy as np
    import loro_b200
    from loro_b200 import api
    blobs = [workloads.make_doc_history(8100 + s, n_sites=3, n_ops=180)[0] for s in range(3)]
    blobs.append(workloads.make_tree_history(8200, n_sites=3, n_base=20, n_ops=70)[0])
    b = loro_b200.import_batch(blobs, flags=api.LB_FLAG_KEEP_DEVICE, lib_path=EMU)
    want = {k: [] for k in ("op_prop", "op_len", "op_counter", "op_vtype", "ch_counter", "ch_len", "ch_lamport", "ch_ts",
                            "dep_counter", "blk_doc", "blk_nchanges")}
    vt_of = {"insert_text": 5, "insert": 11, "map_set": 11, "map_del": 8, "delete": 9, "tree_create": 16, "tree_move": 16, "tree_delete": 16}
    for d, blob in enumerate(blobs):
        for blk in oracle.decode_dump(blob)["blocks"]:
            want["blk_doc"].append(d)
            want["blk_nchanges"].append(blk["n_changes"])
            for ch in blk["changes"]:
                want["ch_counter"].append(ch["counter"])
                want["ch_lamport"].append(ch["lamport"])
                want["ch_ts"].append(ch["timestamp"])
                want["ch_len"].append(ch["ops"][-1]["counter"] + ch["ops"][-1]["len"] - ch["counter"])
                want["dep_counter"] += [c for p, c in ch["deps"] if str(p) != str(ch["peer"])]
                for op in ch["ops"]:
                    want["op_prop"].append(op["prop"])
                    want["op_len"].append(op["len"])
                    want["op_counter"].append(op["counter"])
                    want["op_vtype"].append(vt_of[op["kind"]])
    for name, w in want.items():
        got = b.debug_table(name)
        assert len(got) == len(w), (name, len(got), len(w))
        assert np.array_equal(np.asarray(got, dtype=np.int64), np.asarray(w, dtype=np.int64)), name


@pytest.mark.parametrize("seed", range(4))
def test_partially_known_changes_are_trimmed(seed):
    """import_batch of two blobs whose changes overlap in the middle of an op (oplog.rs:181-196, change.rs:203-258):
    the known head is trimmed on import; state, version, export(all_updates) and export(updates(vv)) equal the oracle's
    for both arrival orders."""
    import loro_b200
    from loro_b200 import api
    e1, e2, n = workloads.overlapping_update_blobs(seed)
    assert n > 0
    for blobs in ([e1, e2], [e2, e1]):
        ref = OracleDoc(7)
        for bl in workloads.import_batch_order(blobs):
            ref.import_(bl)
        bt = loro_b200.import_batch(blobs, doc_ids=[1, 1], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
        assert bt.status(0).code == 0
        assert bt.json_bytes(0) == ref.json_text()
        assert bt.oplog_vv(0) == ref.oplog_vv()
        assert bt.export_updates(0) == ref.export_updates()
        frm = {p: c // 2 for p, c in ref.oplog_vv().items()}
        assert bt.export_updates(0, frm) == ref.export_updates(frm)


def test_snapshot_blobs_and_unknown_modes():
    """Header checks in the reference's order (encoding.rs:299-330): the checksum of a known mode is verified first, an
    intact FastSnapshot (mode 3) is reported as outside this path (code 5), an unknown mode as incompatible (code 3)."""
    import struct
    import loro_b200
    a = OracleDoc(1)
    a.text_insert(a.get_text("t"), 0, "abc")
    good = a.export_updates()

    def with_mode(blob, mode, reseal=True):
        b = bytearray(blob)
        b[20], b[21] = mode >> 8, mode & 255
        if reseal:
            h = oracle.i64s(oracle.codec("xxh32", bytes(b[20:]), 0x4F524F4C))[0] & 0xFFFFFFFF
            b[16:20] = struct.pack("<I", h)
        return bytes(b)
    snap_ok, snap_bad, future = with_mode(good, 3), with_mode(good, 3, reseal=False), with_mode(good, 9)
    b = loro_b200.import_batch([snap_ok, snap_bad, future, good], lib_path=EMU)
    assert [b.status(i).code for i in range(4)] == [5, 2, 3, 0]


@pytest.mark.parametrize("seed", range(6))
def test_import_batch_status_of_overlapping_updates(seed):
    """ImportStatus of import_batch over blobs that overlap, repeat, arrive out of causal order or miss a part: the
    engine's per-document status must equal the reference's fold of per-blob statuses (loro.rs:1228-1258) -- success
    starts, pending hulls of changes parked by a blob's first pass even when a later blob releases them."""
    import random
    import loro_b200
    rng = random.Random(9000 + seed)
    blob, js, tot, sites = workloads.make_doc_history(4200 + seed, n_sites=2 + seed % 3, n_ops=160 + 30 * seed)
    full = sites[0]
    blobs = []
    for _ in range(3 + seed % 3):
        lo = {p: rng.randrange(0, c + 1) for p, c in tot.items() if rng.random() < 0.8}
        blobs.append(full.export_updates(lo))
    for p in list(tot)[:2]:
        blobs.append(full.export_updates({q: c for q, c in tot.items() if q != p}))   # one peer's changes only
    rng.shuffle(blobs)
    if seed % 2:
        blobs.append(blobs[0])
    ref = OracleDoc(31)
    ost = ref.import_batch(blobs)
    r = loro_b200.import_batch(blobs, doc_ids=[3] * len(blobs), lib_path=EMU)
    st = r.status(0)
    assert r.n_docs == 1 and st.code == 0
    assert r.json_bytes(0) == ref.json_text()
    assert r.oplog_vv(0) == ref.oplog_vv()
    assert st.success == ost["success"] and st.pending == ost["pending"], (st, ost)


def test_host_batch_split_into_overlapping_sub_batches():
    """import_batch(split=k): consecutive sub-batches, two C-ABI calls in flight; every accessor answers as the
    unsplit batch does (documents are independent)."""
    import loro_b200
    from loro_b200 import api
    blobs = [workloads.make_doc_history(6100 + i, n_sites=2 + i % 2, n_ops=50 + 7 * i)[0] for i in range(11)]
    one = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU, split=1)
    many = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU, split=3)
    assert isinstance(many, api.MultiBatch) and many.n_docs == one.n_docs == 11
    many.fetch_json()
    many.fetch_exports()
    for i in range(11):
        assert many.status(i) == one.status(i)
        assert many.json_bytes(i) == one.json_bytes(i)
        assert many.oplog_vv(i) == one.oplog_vv(i) and many.oplog_frontiers(i) == one.oplog_frontiers(i)
        assert many.export_updates(i) == one.export_updates(i)
    a, b = many.counters(), one.counters()
    assert a["atom_ops"] == b["atom_ops"] and a["state_hash"] == b["state_hash"] and a["docs_ok"] == 11
    assert api.auto_split(blobs) == 1


@pytest.mark.parametrize("mode", ["warp"])
def test_alternative_decoders_stay_parity_green(mode):
    """The decoder that is not the default (LB_DECODE=warp: TMA-staged, a warp per block, faster on tree-move batches
    and slower on list / map batches -- DESIGN.md section 4) is kept buildable and correct: same JSON, status and
    exported bytes as the oracle on mixed, tree and large-insert documents, through its lane-parallel fast path and
    through the one-lane fallback it shares with the default decoder."""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from tests import workloads\n"
        "from tests.engine_checks import check_batch_against_oracle\n"
        "from tests.export_checks import check_export_against_oracle\n"
        "import loro_b200\n"
        "blobs = [workloads.make_doc_history(8100 + i, n_sites=3, n_ops=180)[0] for i in range(5)]\n"
        "blobs.append(workloads.make_tree_history(11, n_sites=3, n_base=25, n_ops=70)[0])\n"
        "b = check_batch_against_oracle(blobs, lib_path=%r)\n"
        "t = b.timings()\n"
        "check_export_against_oracle(blobs[:3], lib_path=%r)\n"
        "print('ok', t['decode_fast_blocks'], t['decode_lane_blocks'], t['decode_unstaged_blocks'])\n"
    ) % (os.path.dirname(HERE), EMU, EMU)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, LB_DECODE=mode), capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-1500:]
    fast, lane = int(out.stdout.split()[1]), int(out.stdout.split()[2])
    assert fast > 0, out.stdout     # the staged decoder really took its fast path
    assert lane > 0, out.stdout     # ... and its one-lane fallback (decode_block_rows_cols) on some staged blocks
