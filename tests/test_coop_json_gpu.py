"""State JSON of List and Text containers with many runs (written 32 pieces at a time) on the H100 (the CUDA build),
against the reference byte for byte: the emulated suite's documents."""
import pytest

from . import coop_json_checks as cj

pytestmark = pytest.mark.gpu


def test_many_run_containers():
    cj.check()
