"""Phase 7 (re-export) on the H100 (the CUDA build) with staging slots smaller than the blocks need: the cases of
tests/export_staging_checks.py, the same as test_export_staging_emu.py.  These batches are small, so they reach the
unbounded encoder; test_large_batch_gpu.py sends blocks of the bounded build through the retry."""
import pytest

from tests import export_staging_checks as sc
from tests.export_staging_checks import stage_cap  # noqa: F401 -- the fixture

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [21, 22])
def test_every_block_outgrows_its_slot_random_histories(stage_cap, seed):
    sc.every_block_outgrows_random_histories(stage_cap, seed)


def test_some_blocks_outgrow_their_slot_random_histories(stage_cap):
    sc.some_blocks_outgrow_random_histories(stage_cap)


def test_every_block_outgrows_its_slot_generator_documents(stage_cap):
    sc.every_block_outgrows_generator_documents(stage_cap)


def test_every_block_outgrows_its_slot_split_changes_and_trace(stage_cap, golden_dir):
    sc.every_block_outgrows_split_changes_and_trace(stage_cap, golden_dir)


@pytest.mark.parametrize("cap", [0, 1000])
def test_slot_overflow_export_from_version_vector(stage_cap, cap):
    sc.slot_overflow_export_from_version_vector(stage_cap, cap)
