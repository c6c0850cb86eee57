"""Malformed input must never make a kernel read or write outside its tables: mutation fuzzing of the emulated
kernels with guard pages around every device allocation (tests/tools/fuzz_emu.py)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.mark.parametrize("seed,wide,decode", [
    pytest.param(21, False, None, id="21-False"),
    pytest.param(23, False, None, id="23-False"),
    pytest.param(61, True, None, id="61-True"),
    pytest.param(61, True, "warp", id="61-True-warp"),   # the warp decoder: fast path, one-lane fallback, unstaged blocks
])
def test_mutated_blobs_stay_inside_their_tables(seed, wide, decode):
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])
    env = dict(os.environ, LB_EMU_GUARD="1", LB_EMU_THREADS="1")
    if decode:
        env["LB_DECODE"] = decode
    if wide:
        env["LB_FUZZ_WIDE"] = "1"   # more document shapes (seed 61 used to find a list insert whose item count lied)
    out = subprocess.run([sys.executable, os.path.join(HERE, "tools", "fuzz_emu.py"), EMU, str(seed), "150"],
                         env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "fuzz done 150" in out.stdout


def test_mutated_updates_among_overlapping_blobs_of_one_document():
    """import_batch groups and docset imports where one of several overlapping updates is damaged (and re-sealed): copy
    selection, applied-order lists, per-copy epochs and the export of multi-blob documents on inconsistent input"""
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])
    env = dict(os.environ, LB_EMU_GUARD="1", LB_EMU_THREADS="1", LB_FUZZ_MULTI="1")
    out = subprocess.run([sys.executable, os.path.join(HERE, "tools", "fuzz_emu.py"), EMU, "77", "80"],
                         env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "fuzz done 80" in out.stdout
