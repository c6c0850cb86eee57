"""Phase 7 (re-export) on the emulated kernels: byte parity with the oracle's export of the same document."""
import os
import subprocess

import pytest

from oracle import OracleDoc
from tests import workloads
from tests.export_checks import check_export_against_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def test_export_small_mixed_doc():
    a = OracleDoc(1)
    t = a.get_text("text"); a.text_insert(t, 0, "Hello"); a.text_insert(t, 5, " World")
    l = a.get_list("list"); a.list_insert(l, 0, 1, 2, 3); a.delete(l, 1, 1)
    m = a.get_map("map"); a.map_set(m, "k", 5); a.map_set(m, "z", "str"); a.map_delete(m, "k")
    check_export_against_oracle([a.export_updates()], lib_path=EMU)


@pytest.mark.parametrize("seed", [11, 12, 13, 14])
def test_export_random_multi_site_histories(seed):
    blobs = [workloads.make_doc_history(seed * 100 + i, n_sites=2 + i % 4, n_ops=200 + 40 * i, sync_prob=0.03 + 0.02 * (i % 3))[0]
             for i in range(8)]
    check_export_against_oracle(blobs, lib_path=EMU)


def test_export_generator_documents():
    from loro_b200.workload import C3Batch
    gen = C3Batch(6, n_ops=2500, threads=4)
    check_export_against_oracle(gen.blobs(), lib_path=EMU)


def test_export_split_changes_and_trace(golden_dir):
    """Changes above MAX_BLOCK_SIZE enter the store in segments (split_change_then_insert): the 1,000-op prefix
    change of full-size C3 documents, and the merged typing runs of the automerge trace."""
    import gzip
    from loro_b200.workload import C3Batch
    blobs = C3Batch(2, n_ops=10000, threads=2).blobs()
    blobs.append(gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read())
    check_export_against_oracle(blobs, lib_path=EMU, reimport=False)


def test_export_typing_runs_merge_across_changes():
    """Consecutive inserts / deletes in separate commits: stored changes merge (same timestamp is not required for
    ops inside one change; across changes can_merge_right needs ts_b <= ts_a) and op runs re-merge on export."""
    a = OracleDoc(7)
    t = a.get_text("t")
    for i, ch in enumerate("the quick brown fox"):
        a.text_insert(t, i, ch)
        if i % 3 == 2:
            a.commit()
    l = a.get_list("l")
    for i in range(40):
        a.list_insert(l, i, i)
    a.commit()
    for i in range(10):
        a.delete(l, 5, 1)          # forward deletes at one position merge into one span
    for i in range(10):
        a.delete(l, 20 - i, 1)     # backward deletes merge with a negative length
    a.commit()
    check_export_against_oracle([a.export_updates()], lib_path=EMU)


def test_export_needs_flag():
    import loro_b200
    from loro_b200 import api
    b = OracleDoc(4)
    b.text_insert(b.get_text("t"), 0, "ok")
    plain = loro_b200.import_batch([b.export_updates()], lib_path=EMU)
    with pytest.raises(api.EngineError):
        plain.export_updates(0)


def big_insert_documents():
    """Changes with inserts larger than a block: split_change_then_insert cuts the op itself (Op::slice); the pieces
    re-merge in the store when they are alone and stay apart when other ops follow."""
    import random
    docs = []
    a = OracleDoc(3); a.text_insert(a.get_text("t"), 0, "x" * 6000); docs.append(a)
    a = OracleDoc(3); a.text_insert(a.get_text("t"), 0, "h\u00e9llo w\u00f6rld \U0001F600 " * 900); docs.append(a)
    a = OracleDoc(3); a.list_insert(a.get_list("l"), 0, *list(range(3000))); docs.append(a)
    a = OracleDoc(3); t = a.get_text("t"); a.text_insert(t, 0, "abc"); a.text_insert(t, 1, "y" * 9000)
    a.text_insert(t, 5, "zz"); a.map_set(a.get_map("m"), "k", 1); docs.append(a)
    a = OracleDoc(3); l = a.get_list("l"); a.list_insert(l, 0, *["s%d" % i for i in range(1500)])
    a.list_insert(l, 3, *[7] * 1200); docs.append(a)
    a = OracleDoc(3); t = a.get_text("t"); a.text_insert(t, 0, "p" * 4090); a.text_insert(t, 4090, "r" * 10); a.commit()
    a.text_insert(t, 0, "s" * 8200); docs.append(a)
    for seed in (1, 2):
        a = OracleDoc(3); t = a.get_text("t")
        rnd = random.Random(seed)
        for _ in range(24):
            n = rnd.choice([1, 3, 50, 700, 4093, 4096, 5000, 12000])
            a.text_insert(t, rnd.randrange(0, a.seq_len(t) + 1), "".join(rnd.choice("ab \u00e9\U0001F600") for _ in range(n)))
            if rnd.random() < 0.3:
                a.commit()
            if rnd.random() < 0.3 and a.seq_len(t) > 10:
                a.delete(t, rnd.randrange(0, a.seq_len(t) - 5), rnd.randrange(1, 5))
        docs.append(a)
    return [d.export_updates() for d in docs]


def test_export_inserts_larger_than_a_block():
    check_export_against_oracle(big_insert_documents(), lib_path=EMU)


def test_export_regrows_the_segment_tables(monkeypatch, golden_dir):
    """LB_EXPORT_TIGHT_SEGCAP sizes the segment / final-change tables for one segment per change: every workload whose
    changes enter the store in several segments then takes the path that grows them after pass 0."""
    import gzip
    from loro_b200.workload import C3Batch
    monkeypatch.setenv("LB_EXPORT_TIGHT_SEGCAP", "1")
    check_export_against_oracle(big_insert_documents(), lib_path=EMU)
    blobs = C3Batch(2, n_ops=10000, threads=2).blobs()
    blobs.append(gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read())
    check_export_against_oracle(blobs, lib_path=EMU, reimport=False)


def test_export_with_pending_changes_and_after_import_batch():
    """Pending changes stay out of the export but their payloads still moved the arenas; a document built from
    several blobs is exported as the reference would after import_batch (blobs sorted by change count first)."""
    import random
    import loro_b200
    import oracle
    from loro_b200 import api
    from tests.test_engine_emu import _per_peer_blobs

    def change_num(blob):
        return sum(b["n_changes"] for b in oracle.decode_dump(blob)["blocks"])

    for seed in range(3300, 3306):
        whole, js, tot, parts = _per_peer_blobs(seed, n_sites=3, n_ops=200)
        # one per-peer blob alone: whatever depends on the other peers stays pending
        b = loro_b200.import_batch(parts, flags=api.LB_FLAG_EXPORT, lib_path=EMU)
        for i, p in enumerate(parts):
            ref = OracleDoc(5)
            ref.import_(p)
            assert b.export_updates(i) == ref.export_updates(), (seed, i)
        # all of them into one document, shuffled, sometimes with a duplicate
        random.Random(seed).shuffle(parts)
        if seed % 2:
            parts.append(parts[0])
        ref = OracleDoc(5)
        for p in sorted(parts, key=lambda p: -change_num(p)):    # loro.rs:1198-1202 (stable)
            ref.import_(p)
        g = loro_b200.import_batch(parts, doc_ids=[1] * len(parts), flags=api.LB_FLAG_EXPORT, lib_path=EMU)
        assert g.json_bytes(0) == ref.json_text()
        assert g.export_updates(0) == ref.export_updates(), seed


@pytest.mark.parametrize("seed", range(3))
def test_export_from_version_vector(seed):
    """lb_doc_export_updates(from): Change::slice / Op::slice at arbitrary cut points (text incl. multi-byte UTF-8, list
    items, delete spans in both directions, nested values, child containers)."""
    from tests.export_checks import check_export_from_versions
    blob = workloads.make_doc_history(7000 + seed, n_sites=2 + seed, n_ops=220)[0]
    check_export_from_versions(blob, lib_path=EMU, seed=seed)


def test_c1_driven_by_the_engine():
    """BASELINE config C1 end to end: A and B each insert into a List; A's side of the sync -- export(updates(vv_B)) --
    comes out of the engine byte-identical to the reference path's, and B converges after importing it."""
    import random
    import loro_b200
    from loro_b200 import api
    rnd = random.Random(3)
    a, b = OracleDoc(1), OracleDoc(2)
    la, lb = a.get_list("list"), b.get_list("list")
    for k in range(150):
        a.list_insert(la, rnd.randint(0, a.seq_len(la)), rnd.randint(-10**6, 10**6))
        b.list_insert(lb, rnd.randint(0, b.seq_len(lb)), rnd.randint(-10**6, 10**6))
        if k % 10 == 9:
            a.commit(); b.commit()
    workloads.merge(a, b)                                  # A now holds both histories
    batch = loro_b200.import_batch([a.export_updates()], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    update_for_b = batch.export_updates(0, b.oplog_vv())
    assert update_for_b == a.export_updates(b.oplog_vv())
    b.import_(update_for_b)
    assert b.json_text() == a.json_text() == batch.json_bytes(0)


def test_export_from_cut_inside_pasted_inserts_and_trees():
    from tests.export_checks import check_export_from_versions
    big = OracleDoc(9)
    big.text_insert(big.get_text("t"), 0, "wé " * 2500)           # one insert, several blocks
    big.list_insert(big.get_list("l"), 0, *list(range(1500)))
    big.commit()
    big.text_insert(big.get_text("t"), 10, "tail")
    check_export_from_versions(big.export_updates(), lib_path=EMU, seed=1)
    check_export_from_versions(workloads.make_tree_history(31, n_sites=3, n_base=25, n_ops=90, mixed=True)[0], lib_path=EMU, seed=2)
