"""Phase 7's per-change row pass on the H100 (the CUDA build) against the oracle's export: the change shapes of
tests/change_rows_checks.py on the 32-row chunk boundaries, the same cases as test_export_change_rows_emu.py.  On the
device the lanes of a warp run concurrently, so the delete runs and text runs carried across chunks on shuffled
registers are checked where the emulator, which switches lanes only at warp collectives, cannot reorder them."""
import pytest

from tests import change_rows_checks as cr
from tests.export_checks import check_export_against_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_rows", cr.CHUNK_ROW_COUNTS)
def test_changes_of_chunk_sized_row_counts(n_rows):
    check_export_against_oracle(cr.chunk_sized_row_counts(n_rows))


@pytest.mark.parametrize("lead", cr.TEXT_RUN_LEADS)
@pytest.mark.parametrize("pad", cr.TEXT_RUN_PADS)
def test_text_runs_placed_on_chunk_boundaries(pad, lead):
    check_export_against_oracle(cr.text_runs_on_chunk_boundaries(pad, lead))


def test_string_generation_changes_inside_a_run():
    check_export_against_oracle(cr.string_generation_runs())


@pytest.mark.parametrize("n", cr.DELETE_CHAIN_LENGTHS)
def test_single_element_delete_chains_both_directions(n):
    check_export_against_oracle(cr.delete_chains(n))


def test_trimmed_changes():
    cr.check_trimmed_changes()


def test_change_over_the_block_size():
    check_export_against_oracle(cr.change_over_the_block_size())


# ---- rows of one change that merge only on import


@pytest.mark.parametrize("n", cr.MERGE_DELETE_LENGTHS)
@pytest.mark.parametrize("lead", cr.MERGE_DELETE_LEADS)
def test_single_element_deletes_merge_into_directed_spans(n, lead):
    check_export_against_oracle(cr.deletes_merge_into_directed_spans(n, lead))


def test_delete_runs_of_several_spans():
    check_export_against_oracle(cr.delete_runs_of_several_spans())


@pytest.mark.parametrize("lead", cr.MERGE_RUN_LEADS)
@pytest.mark.parametrize("pad", cr.MERGE_RUN_PADS)
def test_text_and_list_runs_merge_across_chunks(pad, lead):
    check_export_against_oracle(cr.text_and_list_runs_across_chunks(pad, lead))


@pytest.mark.parametrize("seed", cr.PIECE_SEEDS)
def test_random_histories_in_pieces(seed):
    check_export_against_oracle(cr.random_histories_in_pieces(seed))


def test_change_over_the_block_size_in_pieces():
    check_export_against_oracle(cr.change_over_the_block_size_in_pieces())
