"""Shared parity checks: the engine (real CUDA library, or the emulated test build) against the oracle."""
import json

import oracle
from oracle import OracleDoc

import loro_b200


def check_batch_against_oracle(blobs, lib_path=None, expect_json=None):
    """Import `blobs` as one batch; compare every document with a fresh oracle doc importing the same blob."""
    batch = loro_b200.import_batch(blobs, lib_path=lib_path)
    assert batch.n_docs == len(blobs)
    for i, blob in enumerate(blobs):
        o = OracleDoc(1)
        try:
            ost = o.import_(blob)
            ocode = 0
        except oracle.ImportError_ as e:
            ocode = e.code
        st = batch.status(i)
        if ocode:
            # oracle codes: 1 short, 2 magic, 3 checksum, 4 mode, 10 decode, 11 snapshot mode
            want = {1: 1, 2: 1, 3: 2, 4: 3, 10: (1, 4), 11: 5}[ocode]
            assert st.code == want or (isinstance(want, tuple) and st.code in want), (i, st, ocode)
            continue
        assert st.code == 0, (i, st)
        assert batch.json_bytes(i) == (expect_json[i] if expect_json else o.json_text()), i
        assert batch.oplog_vv(i) == o.oplog_vv(), i
        assert batch.oplog_frontiers(i) == sorted(o.frontiers()), (i, batch.oplog_frontiers(i), o.frontiers())
        assert st.success == ost["success"], (i, st.success, ost["success"])
        assert st.pending == ost["pending"], (i, st.pending, ost["pending"])
    return batch


def check_c5_documents_of_atoms(atoms, lib_path=None):
    """One batch of config C5 tree documents, document k of atoms[k] atom ops (n_nodes creates + 3 peers x n_moves
    moves, n_moves = 1,000 or a sixth of the atoms): JSON against the generator's own merge and the oracle, re-exported bytes against the oracle's.  The
    largest document decides whether the tree apply keeps its parent links in shared memory (up to
    TREE_S_NODES_MAX = 32,768 atoms, 16-bit links next to the 0xFFFD..0xFFFF sentinels) or, for the documents past
    it, in global memory while the others of the launch keep theirs in shared memory."""
    from loro_b200.workload import C5Batch
    from .export_checks import check_export_against_oracle
    blobs, want = [], []
    for k, a in enumerate(atoms):
        n_moves = min(1000, a // 6)
        g = C5Batch(1, n_nodes=a - 3 * n_moves, n_moves=n_moves, first_doc=k, want_json=True)
        assert g.atom_ops == a, (k, g.atom_ops, a)
        blobs.append(g.blob(0))
        want.append(g.expected_json(0))
        g.close()
    batch = check_batch_against_oracle(blobs, lib_path=lib_path, expect_json=want)
    assert batch.counters()["atom_ops"] == sum(atoms)
    check_export_against_oracle(blobs, lib_path=lib_path, reimport=False)
    return batch
