"""The per-document widths of the warp-per-document kernels on the emulated build: documents of 8 / 9 / 32 / 33 / 64 /
65 peers, trees of 8 to 40 peers with and without meta maps, 31 to 65 containers and keys, ropes of 31 to 32,769
spans and fractional indexes past 32 bytes, through every output against the reference byte for byte, cursors
included (tests/width_checks.py)."""
import os
import subprocess

import pytest

from . import value_checks as vc
from . import width_checks as wc

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


@pytest.fixture(scope="module")
def span_cases():
    """built once: the reference is slow on the 32,769-span rope"""
    return wc.span_cases()


def run(cases):
    for c in cases:
        print(c.name, c.width)
    answers = vc.check_cases(cases, lib_path=EMU)
    wc.check_coverage(cases, answers)


def test_peers():
    run(wc.peer_cases())


def test_trees_and_fractional_indexes():
    run(wc.tree_cases())


def test_containers():
    run(wc.container_cases())


def test_keys():
    run(wc.key_cases())


def test_spans(span_cases):
    run(span_cases)
