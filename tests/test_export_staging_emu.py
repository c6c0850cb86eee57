"""Phase 7 (re-export) on the emulated kernels with staging slots smaller than the blocks need: the cases of
tests/export_staging_checks.py, whose bytes must stay the oracle's whether a block fits its slot or goes through the
retry.  The same cases run on the CUDA build in test_export_staging_gpu.py."""
import os
import subprocess

import pytest

from tests import export_staging_checks as sc
from tests.export_staging_checks import stage_cap  # noqa: F401 -- the fixture

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


@pytest.mark.parametrize("seed", [21, 22])
def test_every_block_outgrows_its_slot_random_histories(stage_cap, seed):
    sc.every_block_outgrows_random_histories(stage_cap, seed, lib_path=EMU)


def test_some_blocks_outgrow_their_slot_random_histories(stage_cap):
    sc.some_blocks_outgrow_random_histories(stage_cap, lib_path=EMU)


def test_every_block_outgrows_its_slot_generator_documents(stage_cap):
    sc.every_block_outgrows_generator_documents(stage_cap, lib_path=EMU)


def test_every_block_outgrows_its_slot_split_changes_and_trace(stage_cap, golden_dir):
    sc.every_block_outgrows_split_changes_and_trace(stage_cap, golden_dir, lib_path=EMU)


@pytest.mark.parametrize("cap", [0, 1000])
def test_slot_overflow_export_from_version_vector(stage_cap, cap):
    sc.slot_overflow_export_from_version_vector(stage_cap, cap, lib_path=EMU)
