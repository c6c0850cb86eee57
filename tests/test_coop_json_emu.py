"""State JSON of List and Text containers with many runs (written 32 pieces at a time) on the emulated build, against
the reference byte for byte: window and slot edges, runs that start inside their op, escapes at run edges, a nested
value after several windows, containers of 63, 64 and 65 runs."""
import os
import subprocess

import pytest

from . import coop_json_checks as cj

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def test_many_run_containers():
    cj.check(lib_path=EMU)
