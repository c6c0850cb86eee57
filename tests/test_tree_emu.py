"""Movable-tree path (SURVEY 8a row a16) of the product's kernels on the SIMT emulator: decode of the positions arena
and RawTreeMove values, the (lamport, peer)-ordered apply with the cycle check, sibling order, hierarchy JSON with
meta maps -- against the oracle, whose tree path is pinned by the reference's known answers
(tests/test_oracle_semantics.py).  The same checks run on the CUDA build in test_engine_gpu.py."""
import os
import subprocess

import pytest

from oracle import OracleDoc
from tests import workloads
from tests.engine_checks import check_batch_against_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def test_tree_known_answer_through_the_engine():
    """crates/loro/tests/loro_rust_test.rs:426-444."""
    d = OracleDoc(1)
    t = d.get_tree("tree")
    root = d.tree_create(t)
    root2 = d.tree_create(t)
    d.tree_move(t, root2, root)
    d.map_set(d.tree_meta(root), "color", "red")
    b = check_batch_against_oracle([d.export_updates()], lib_path=EMU)
    assert b.get_deep_value(0) == {"tree": [
        {"parent": None, "meta": {"color": "red"}, "id": "0@1", "index": 0, "fractional_index": "80", "children": [
            {"parent": "0@1", "meta": {}, "id": "1@1", "index": 0, "children": [], "fractional_index": "80"}]}]}


def test_tree_concurrent_cycle_and_delete():
    a, b = OracleDoc(1), OracleDoc(2)
    ta, tb = a.get_tree("t"), b.get_tree("t")
    x = a.tree_create(ta)
    y = a.tree_create(ta)
    z = a.tree_create(ta, y)
    workloads.merge(b, a)
    a.tree_move(ta, x, y)
    b.tree_move(tb, y, x)       # closes a cycle with the concurrent move: later in (lamport, peer) order, not effected
    b.tree_delete(tb, z)
    a.map_set(a.tree_meta(z), "k", 1)
    workloads.merge(a, b)
    batch = check_batch_against_oracle([a.export_updates(), b.export_updates()], lib_path=EMU)
    v = batch.get_deep_value(0)["t"]
    assert [n["id"] for n in v] == ["1@1"] and [c["id"] for c in v[0]["children"]] == ["0@1"]


@pytest.mark.parametrize("seed", range(4))
def test_tree_random_histories(seed):
    blobs, jsons = [], []
    for k in range(4):
        blob, js, vv, _ = workloads.make_tree_history(seed * 50 + k, n_sites=2 + (seed + k) % 3, n_base=20 + 10 * k,
                                                      n_ops=100 + 30 * k, mixed=(seed + k) % 2 == 0)
        blobs.append(blob)
        jsons.append(js)
    check_batch_against_oracle(blobs, lib_path=EMU, expect_json=jsons)


def test_tree_equal_positions_and_two_trees():
    """Siblings with equal fractional indexes (concurrent appends under one parent) are ordered by (lamport, peer);
    two tree containers in one document keep separate roots."""
    docs = [OracleDoc(10 + i) for i in range(3)]
    ts = [(d.get_tree("a"), d.get_tree("b")) for d in docs]
    r = docs[0].tree_create(ts[0][0])
    docs[0].tree_create(ts[0][1])
    for j in (1, 2):
        workloads.merge(docs[j], docs[0])
    for i, d in enumerate(docs):
        for _ in range(3):
            d.tree_create(ts[i][0], r)       # everybody appends under r: identical positions across peers
            d.tree_create(ts[i][1])
    for _ in range(2):
        for i in range(3):
            for j in range(3):
                if i != j:
                    workloads.merge(docs[i], docs[j])
    check_batch_against_oracle([docs[0].export_updates()], lib_path=EMU)


def test_tree_export_matches_oracle_bytes():
    """Re-export of tree documents (positions arena with common-prefix compression in sorted order, RawTreeMove
    values, the DELETED_TREE_ROOT pseudo peer of deletes) is byte-identical to the oracle's and round-trips."""
    from tests.export_checks import check_export_against_oracle
    d = OracleDoc(1)
    t = d.get_tree("tree")
    root = d.tree_create(t)
    root2 = d.tree_create(t)
    d.tree_move(t, root2, root)
    d.map_set(d.tree_meta(root), "color", "red")
    d.tree_delete(t, root2)
    blobs = [d.export_updates()]
    for seed in range(5):
        blobs.append(workloads.make_tree_history(900 + seed, n_sites=2 + seed % 3, n_base=25, n_ops=120, mixed=seed % 2 == 0)[0])
    check_export_against_oracle(blobs, lib_path=EMU)


def test_tree_many_nodes_several_blocks_per_peer():
    """A tree large enough for several change blocks per peer (8 estimated bytes per op, 4 KB blocks): block-local
    position registers, positions shared between blocks, long sibling lists (the warp-sorted path)."""
    from tests.export_checks import check_export_against_oracle
    import random
    rnd = random.Random(4)
    a, b = OracleDoc(21), OracleDoc(22)
    ta, tb = a.get_tree("tree"), b.get_tree("tree")
    nodes = []
    for i in range(700):
        parent = rnd.choice(nodes) if nodes and rnd.random() < 0.7 else None
        nodes.append(a.tree_create(ta, parent, -1 if rnd.random() < 0.6 else 0))
        if i % 7 == 0:
            a.commit()
    workloads.merge(b, a)
    for d, t in ((a, ta), (b, tb)):
        for _ in range(250):
            workloads.random_tree_edit(rnd, d, t, p_create=0.2)
    workloads.merge(a, b)
    workloads.merge(b, a)
    assert a.json_text() == b.json_text()
    blob = a.export_updates()
    check_batch_against_oracle([blob], lib_path=EMU)
    check_export_against_oracle([blob], lib_path=EMU)


def test_config_c5_generator_documents():
    """Config C5 shape from the workload generator (its own encoder, its own merge): generator == oracle == kernels,
    for state and for re-exported bytes."""
    from loro_b200.workload import C5Batch
    from tests.export_checks import check_export_against_oracle
    g = C5Batch(5, n_nodes=400, n_moves=120, want_json=True)
    blobs = g.blobs()
    for i, blob in enumerate(blobs):
        o = OracleDoc(1)
        o.import_(blob)
        assert o.json_text() == g.expected_json(i)
        assert o.export_updates() == blob
    check_batch_against_oracle(blobs, lib_path=EMU, expect_json=[g.expected_json(i) for i in range(5)])
    check_export_against_oracle(blobs, lib_path=EMU)


def test_tree_long_sibling_list_with_equal_positions():
    """More than 32 children under one parent, appended concurrently by three peers (equal fractional indexes
    across peers): the warp-sorted sibling path, ties broken by (lamport, peer)."""
    docs = [OracleDoc(30 + i) for i in range(3)]
    ts = [d.get_tree("t") for d in docs]
    r = docs[0].tree_create(ts[0])
    for j in (1, 2):
        workloads.merge(docs[j], docs[0])
    for i, d in enumerate(docs):
        for _ in range(20):
            d.tree_create(ts[i], r)
    for _ in range(2):
        for i in range(3):
            for j in range(3):
                if i != j:
                    workloads.merge(docs[i], docs[j])
    b = check_batch_against_oracle([docs[0].export_updates()], lib_path=EMU)
    assert len(b.get_deep_value(0)["t"][0]["children"]) == 60


def test_tree_links_in_shared_memory_at_their_limit():
    """The largest document has exactly TREE_S_NODES_MAX = 32,768 atoms: every document of the launch keeps its
    16-bit parent links in shared memory, with links up to 32,767 next to the 0xFFFD..0xFFFF sentinels."""
    from tests.engine_checks import check_c5_documents_of_atoms
    check_c5_documents_of_atoms([32768, 760], lib_path=EMU)


def test_tree_links_in_global_memory_past_the_limit():
    """Documents of 32,769 and 36,000 atoms keep their parent links in global memory, while a 32,768-atom and a
    small document of the same launch use 64 KB of shared memory per CTA."""
    from tests.engine_checks import check_c5_documents_of_atoms
    check_c5_documents_of_atoms([32769, 760, 36000, 32768], lib_path=EMU)
