"""Value edges and deep nesting on the H100 (the CUDA build): the emulated suite's documents against the reference byte
for byte through every output, through the default and the warp decoder; one level past LB_MAX_NESTING is
LB_DOC_ERR_UNSUPPORTED on every path."""
import os
import subprocess
import sys

import pytest

from . import value_checks as vc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_value_edges():
    vc.check_cases(vc.scalar_cases() + vc.composite_cases() + vc.warp_edge_cases())


def test_nesting_at_and_past_the_bound():
    vc.check_cases(vc.depth_cases(vc.NEST))
    vc.check_past_bound(vc.depth_cases(vc.NEST + 1))


def test_warp_decoder_fast_path_and_fallback():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "import loro_b200\n"
        "from tests import value_checks as vc\n"
        "cases = vc.warp_edge_cases() + vc.scalar_cases() + vc.depth_cases(vc.NEST)\n"
        "vc.check_cases(cases)\n"
        "vc.check_past_bound(vc.depth_cases(vc.NEST + 1))\n"
        "t = loro_b200.import_batch([c.blob for c in cases]).timings()\n"
        "print('ok', t['decode_fast_blocks'], t['decode_lane_blocks'])\n"
    ) % os.path.dirname(HERE)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, LB_DECODE="warp"), capture_output=True,
                         text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    fast, lane = (int(x) for x in out.stdout.split()[-2:])
    assert fast > 0 and lane > 0, out.stdout
