"""Phase 7 on the emulated kernels: the per-change row pass (a warp per change, 32 rows at a time) against the oracle's
export, on the change shapes of tests/change_rows_checks.py that sit on its 32-row chunk boundaries.  The same cases
run on the CUDA build in test_export_change_rows_gpu.py."""
import os
import subprocess

import pytest

from tests import change_rows_checks as cr
from tests.export_checks import check_export_against_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


@pytest.mark.parametrize("n_rows", cr.CHUNK_ROW_COUNTS)
def test_changes_of_chunk_sized_row_counts(n_rows):
    check_export_against_oracle(cr.chunk_sized_row_counts(n_rows), lib_path=EMU)


@pytest.mark.parametrize("lead", cr.TEXT_RUN_LEADS)
@pytest.mark.parametrize("pad", cr.TEXT_RUN_PADS)
def test_text_runs_placed_on_chunk_boundaries(pad, lead):
    check_export_against_oracle(cr.text_runs_on_chunk_boundaries(pad, lead), lib_path=EMU)


def test_string_generation_changes_inside_a_run():
    check_export_against_oracle(cr.string_generation_runs(), lib_path=EMU)


@pytest.mark.parametrize("n", cr.DELETE_CHAIN_LENGTHS)
def test_single_element_delete_chains_both_directions(n):
    check_export_against_oracle(cr.delete_chains(n), lib_path=EMU)


def test_trimmed_changes():
    cr.check_trimmed_changes(lib_path=EMU)


def test_change_over_the_block_size():
    check_export_against_oracle(cr.change_over_the_block_size(), lib_path=EMU)


# ---- rows of one change that merge only on import


@pytest.mark.parametrize("n", cr.MERGE_DELETE_LENGTHS)
@pytest.mark.parametrize("lead", cr.MERGE_DELETE_LEADS)
def test_single_element_deletes_merge_into_directed_spans(n, lead):
    check_export_against_oracle(cr.deletes_merge_into_directed_spans(n, lead), lib_path=EMU)


def test_delete_runs_of_several_spans():
    check_export_against_oracle(cr.delete_runs_of_several_spans(), lib_path=EMU)


@pytest.mark.parametrize("lead", cr.MERGE_RUN_LEADS)
@pytest.mark.parametrize("pad", cr.MERGE_RUN_PADS)
def test_text_and_list_runs_merge_across_chunks(pad, lead):
    check_export_against_oracle(cr.text_and_list_runs_across_chunks(pad, lead), lib_path=EMU)


@pytest.mark.parametrize("seed", cr.PIECE_SEEDS)
def test_random_histories_in_pieces(seed):
    check_export_against_oracle(cr.random_histories_in_pieces(seed), lib_path=EMU)


def test_change_over_the_block_size_in_pieces():
    check_export_against_oracle(cr.change_over_the_block_size_in_pieces(), lib_path=EMU)
