"""Host-side checks that need no GPU: the C-ABI library builds for sm_90a, loads, exports every symbol the
header declares, and fails loudly (no CPU fallback) when there is no CUDA device."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    path = g.build_engine()
    return ctypes.CDLL(path)


def test_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "loro_b200.h")).read()
    names = set(re.findall(r"\b(lb_[a-z_]+)\s*\(", hdr))
    assert {"lb_import_batch", "lb_import_batch_device", "lb_doc_status", "lb_doc_json", "lb_doc_vv",
            "lb_batch_counters", "lb_batch_timings", "lb_batch_free", "lb_doc_count", "lb_last_error",
            "lb_doc_frontiers", "lb_doc_export_updates", "lb_docset_new", "lb_docset_import", "lb_docset_free"} <= names
    for n in names:
        assert hasattr(lib, n), n


def test_no_cpu_fallback_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    import loro_b200
    with pytest.raises(loro_b200.EngineUnavailable):
        loro_b200.import_batch([b"loro" + bytes(30)])
    with pytest.raises(loro_b200.EngineUnavailable):
        loro_b200.DocSet()


def test_sass_is_sm90a(lib):
    import subprocess
    import loro_b200
    out = subprocess.run(["cuobjdump", "-lelf", loro_b200.library_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out, out


def test_ctypes_structs_match_the_header(tmp_path):
    """api.py's ctypes mirrors of lb_timings, lb_counters and lb_options have the size and field offsets the C compiler
    gives the header's structs; a field api.py names that the header lacks fails the compile."""
    import subprocess
    from loro_b200 import api
    structs = {"lb_timings": api._Timings, "lb_counters": api._Counters, "lb_options": api._Options}
    want, lines = {}, ["#include <stddef.h>", "#include <stdio.h>", '#include "loro_b200.h"', "int main(void) {"]
    for cname, py in structs.items():
        want[cname] = ctypes.sizeof(py)
        lines.append(f'    printf("{cname} %zu\\n", sizeof({cname}));')
        for f, _ in py._fields_:
            want[f"{cname}.{f}"] = getattr(py, f).offset
            lines.append(f'    printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));')
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text("\n".join(lines + ["    return 0;", "}"]) + "\n")
    cc = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe],
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    assert {k: int(v) for k, v in got.items()} == want


def test_plain_c_caller_compiles_links_and_fails_loudly_without_a_device(lib, tmp_path):
    """include/loro_b200.h is plain C (no torch / C++ types in the signatures): examples/c/import_and_docset.c builds
    with -std=c99 -Wall -Wextra -Werror, links against the library and, without a CUDA device, gets LB_ERR_NO_DEVICE."""
    import subprocess
    import loro_b200
    exe = str(tmp_path / "demo")
    libdir = os.path.dirname(loro_b200.library_path())
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "c", "import_and_docset.c"), "-L" + libdir, "-lloro_b200", "-o", exe])
    import torch
    if torch.cuda.is_available():
        return
    out = subprocess.run([exe, os.path.join(ROOT, "tests", "golden", "gv1_update.bin")], capture_output=True, text=True,
                         env=dict(os.environ, LD_LIBRARY_PATH=libdir))
    assert out.returncode == 1 and "no CUDA device" in out.stderr, (out.returncode, out.stderr)
