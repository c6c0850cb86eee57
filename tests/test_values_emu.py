"""Value edges and deep nesting on the emulated build: every output of documents holding i64 / f64 / string / binary
edge values, wide nested maps, container values, the warp decoder's size edges and nesting at LB_MAX_NESTING, against
the reference byte for byte; one level past the bound is LB_DOC_ERR_UNSUPPORTED on every path."""
import os
import subprocess
import sys

import pytest

from . import value_checks as vc

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


def test_scalar_edges():
    vc.check_cases(vc.scalar_cases(), lib_path=EMU)


def test_wide_maps_and_container_values():
    vc.check_cases(vc.composite_cases(), lib_path=EMU)


def test_warp_decoder_size_edges():
    vc.check_cases(vc.warp_edge_cases(), lib_path=EMU)


def test_nesting_at_the_bound():
    vc.check_cases(vc.depth_cases(vc.NEST), lib_path=EMU)


def test_nesting_past_the_bound_is_unsupported():
    vc.check_past_bound(vc.depth_cases(vc.NEST + 1), lib_path=EMU)


def test_warp_decoder_fast_path_and_fallback():
    """LB_DECODE=warp (read once per process, hence the subprocess): the decode-sensitive cases through the warp
    decoder's lane-parallel path and its one-lane fallback, with the same outputs; past the bound still UNSUPPORTED"""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "import loro_b200\n"
        "from tests import value_checks as vc\n"
        "cases = vc.warp_edge_cases() + vc.scalar_cases()[:4] + vc.depth_cases(vc.NEST)[3:5]\n"
        "vc.check_cases(cases, lib_path=%r)\n"
        "vc.check_past_bound(vc.depth_cases(vc.NEST + 1)[3:5], lib_path=%r)\n"
        "t = loro_b200.import_batch([c.blob for c in cases], lib_path=%r).timings()\n"
        "print('ok', t['decode_fast_blocks'], t['decode_lane_blocks'])\n"
    ) % (os.path.dirname(HERE), EMU, EMU, EMU)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, LB_DECODE="warp"), capture_output=True,
                         text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    fast, lane = (int(x) for x in out.stdout.split()[-2:])
    assert fast > 0 and lane > 0, out.stdout
