"""Phase 5 hands documents to warps from a queue: one warp integrates many documents one after another, and nothing of
one document may leak into the next through the warp's shared-memory state.  The emulated launch is a single CTA of
four warps, so every warp here runs several of the documents below, healthy ones right after ones the kernel skips."""
import os
import subprocess

import pytest

from tests import workloads
from tests.engine_checks import check_batch_against_oracle
from tests.export_checks import check_export_against_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def _healthy():
    from loro_b200.workload import C3Batch
    docs = C3Batch(3, n_ops=2000, threads=2).blobs()
    for k in range(6):
        docs.append(workloads.make_doc_history(6100 + k, n_sites=2 + k % 3, n_ops=150 + 30 * k, sync_prob=0.04)[0])
    for k in range(2):   # peers beyond 32: atom bases and tracker versions outside shared memory
        docs.append(workloads.make_doc_history(6200 + k, n_sites=40, n_ops=500, sync_prob=0.04)[0])
    return docs


def test_one_warp_many_documents():
    healthy = _healthy()
    skipped = workloads.skipped_kinds(healthy[0])
    blobs = []
    for i, h in enumerate(healthy):   # every skipped document sits right before a healthy one
        blobs.append(skipped[i % len(skipped)])
        blobs.append(h)
    check_batch_against_oracle(blobs, lib_path=EMU)
    # re-export in one batch too, without the blob the oracle rejects (no round trip: the pending document's export
    # carries no change, so it does not register the container its pending change created)
    check_export_against_oracle([b for i, b in enumerate(blobs) if i % (2 * len(skipped)) != 0], lib_path=EMU,
                                reimport=False)
