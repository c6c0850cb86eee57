"""Phase 7 (re-export) with staging slots smaller than the blocks need, shared by test_export_staging_emu.py and
test_export_staging_gpu.py.

The encoder writes each output block once, into a staging slot sized from the block's rows and store estimate, and
the blobs are assembled from the slots.  A block that outgrows its slot is encoded again by the same code, into a
retry slot of its exact size.  LB_EXPORT_STAGE_CAP caps every first slot's capacity (in bytes): 0 sends every block
through the retry, a small cap only the larger blocks.  Either way the bytes must stay the oracle's.  The library
reads the cap at every export, so a test sets it in its own process."""
import gzip
import os
import re

import pytest

from . import workloads
from .export_checks import check_export_against_oracle, check_export_from_versions

TRACE = re.compile(r"\[trace\] export: (\d+) blocks, (\d+) outgrew their staging slot")


@pytest.fixture
def stage_cap(monkeypatch, capfd):
    """Sets the slot cap; returns a function giving (blocks, blocks that outgrew their slot) over the exports so far."""
    monkeypatch.setenv("LB_PHASE_TRACE", "1")

    def setcap(cap):
        monkeypatch.setenv("LB_EXPORT_STAGE_CAP", str(cap))

    def counts():
        err = capfd.readouterr().err
        m = TRACE.findall(err)
        assert m, "no export trace line"
        return sum(int(a) for a, _ in m), sum(int(b) for _, b in m)
    return setcap, counts


def random_histories(seed):
    return [workloads.make_doc_history(seed * 100 + i, n_sites=2 + i % 4, n_ops=200 + 40 * i, sync_prob=0.03 + 0.02 * (i % 3))[0]
            for i in range(6)]


def every_block_outgrows_random_histories(stage_cap, seed, lib_path=None):
    setcap, counts = stage_cap
    setcap(0)
    check_export_against_oracle(random_histories(seed), lib_path=lib_path)
    blocks, ovf = counts()
    assert blocks > 0 and ovf == blocks


def some_blocks_outgrow_random_histories(stage_cap, lib_path=None):
    setcap, counts = stage_cap
    setcap(1000)
    check_export_against_oracle(random_histories(23), lib_path=lib_path)
    blocks, ovf = counts()
    assert 0 < ovf < blocks, (blocks, ovf)


def every_block_outgrows_generator_documents(stage_cap, lib_path=None):
    from loro_b200.workload import C3Batch
    setcap, counts = stage_cap
    setcap(0)
    check_export_against_oracle(C3Batch(4, n_ops=2500, threads=4).blobs(), lib_path=lib_path)
    blocks, ovf = counts()
    assert blocks > 0 and ovf == blocks


def every_block_outgrows_split_changes_and_trace(stage_cap, golden_dir, lib_path=None):
    from loro_b200.workload import C3Batch
    setcap, counts = stage_cap
    setcap(0)
    blobs = C3Batch(2, n_ops=10000, threads=2).blobs()
    blobs.append(gzip.open(os.path.join(golden_dir, "automerge_trace_blob.bin.gz"), "rb").read())
    check_export_against_oracle(blobs, lib_path=lib_path, reimport=False)
    blocks, ovf = counts()
    assert blocks > 0 and ovf == blocks


def slot_overflow_export_from_version_vector(stage_cap, cap, lib_path=None):
    setcap, counts = stage_cap
    setcap(cap)
    check_export_from_versions(workloads.make_doc_history(7220, n_sites=3, n_ops=260)[0], lib_path=lib_path, seed=1)
    blocks, ovf = counts()
    if cap == 0:
        assert blocks > 0 and ovf == blocks
    else:
        assert 0 < ovf < blocks, (blocks, ovf)
