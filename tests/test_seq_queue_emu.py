"""Phase 5 hands documents to warps from a queue: one warp integrates many documents one after another, and nothing of
one document may leak into the next through the warp's shared-memory state.  The emulated launch is a single CTA of
four warps, so every warp here runs several of the documents below, healthy ones right after ones the kernel skips."""
import os
import subprocess

import pytest

from oracle import OracleDoc
from tests import workloads
from tests.engine_checks import check_batch_against_oracle
from tests.export_checks import check_export_against_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def _pending_only():
    """A document whose one change depends on a change the blob does not carry: nothing of it is applied."""
    a = OracleDoc(5)
    a.text_insert(a.get_text("t"), 0, "abc")
    a.commit()
    vv = a.oplog_vv()
    a.text_insert(a.get_text("t"), 3, "def")
    return a.export_updates(vv)


def _map_only():
    a = OracleDoc(6)
    m = a.get_map("map")
    a.map_set(m, "k", 1)
    a.map_set(m, "s", "v")
    return a.export_updates()


def _bad_checksum(blob):
    return blob[:30] + bytes([blob[30] ^ 1]) + blob[31:]


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
    skipped = [_bad_checksum(healthy[0]), _pending_only(), _map_only(), OracleDoc(8).export_updates()]
    blobs = []
    for i, h in enumerate(healthy):   # every skipped document sits right before a healthy one
        blobs.append(skipped[i % len(skipped)])
        blobs.append(h)
    check_batch_against_oracle(blobs, lib_path=EMU)
    # re-export in one batch too, without the blob the oracle rejects (no round trip: the pending document's export
    # carries no change, so it does not register the container its pending change created)
    check_export_against_oracle([b for i, b in enumerate(blobs) if i % (2 * len(skipped)) != 0], lib_path=EMU,
                                reimport=False)
