"""The per-document widths of the warp-per-document kernels on the H100 (the CUDA build): the emulated suite's documents
(tests/width_checks.py) against the reference byte for byte through every output, cursors included; and config C5
documents at their stated size with 8, 9 and 33 moving peers, which have no meta maps and so take the parallel tree
writer with its shared peer table and without it."""
import pytest

from . import value_checks as vc
from . import width_checks as wc

pytestmark = pytest.mark.gpu


def run(cases):
    for c in cases:
        print(c.name, c.width)
    wc.check_coverage(cases, vc.check_cases(cases))


def test_peers_trees_containers_keys():
    run(wc.peer_cases() + wc.tree_cases() + wc.container_cases() + wc.key_cases())


def test_spans():
    run(wc.span_cases())


@pytest.mark.parametrize("n_peers", [wc.TREE_TXT_PEERS, wc.TREE_TXT_PEERS + 1, wc.WARP + 1])
def test_config_c5_full_size_with_many_peers(n_peers):
    from loro_b200.workload import C5Batch
    from .engine_checks import check_batch_against_oracle
    from .export_checks import check_export_against_oracle
    g = C5Batch(4, n_peers=n_peers, want_json=True)
    blobs = g.blobs()
    want = [g.expected_json(i) for i in range(g.n_docs)]
    g.close()
    for b in blobs:
        ref = wc.reference(b)
        P = len(ref.oplog_vv())
        assert P == n_peers and not any(n["meta"] for n in wc.tree_json_nodes(ref.json_text())), P
        print("C5 n_peers=%d: P=%d" % (n_peers, P))
    check_batch_against_oracle(blobs, expect_json=want)
    check_export_against_oracle(blobs)
