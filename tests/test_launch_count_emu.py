"""lb_timings.kernel_launches on the emulated build: the emulator prints one `simt_emu: launch <kernel>` line per launch
when LB_EMU_KTRACE is set, and the counter of a batch must equal the number of those lines printed on its behalf --
also where a phase skips kernels (no change, no output block), copies stored blobs, or exports on demand later.
And the phase times of a batch come from named events: every one is a finite number >= 0, the empty batch's included."""
import math
import os
import subprocess

import pytest

import loro_b200
from loro_b200 import api
from oracle import OracleDoc
from tests import workloads

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu", "libloro_b200_emu.so")
PHASES = ("h2d", "frame", "decode", "resolve", "classify", "integrate", "tree", "materialise", "reexport", "d2h",
          "total_device")


@pytest.fixture(scope="session", autouse=True)
def build_emu():
    subprocess.check_call([os.path.join(HERE, "emu", "build_emu.sh")])


@pytest.fixture
def launches(monkeypatch, capfd):
    """Switches the launch trace on; returns a function giving the number of launches traced since its last call."""
    monkeypatch.setenv("LB_EMU_KTRACE", "1")
    capfd.readouterr()

    def traced():
        return sum(line.startswith("simt_emu: launch ") for line in capfd.readouterr().err.splitlines())
    return traced


def mixed_documents():
    return [workloads.make_doc_history(4100 + i, n_sites=2 + i % 3, n_ops=120 + 30 * i)[0] for i in range(5)]


def test_counter_equals_traced_launches_mixed_documents_with_export(launches):
    b = loro_b200.import_batch(mixed_documents(), flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    n = launches()
    assert n > 10 and b.timings()["kernel_launches"] == n


def _bad_checksum():
    blob = workloads.make_doc_history(4200, n_sites=2, n_ops=60)[0]
    return blob[:30] + bytes([blob[30] ^ 1]) + blob[31:]


@pytest.mark.parametrize("blob", [lambda: OracleDoc(3).export_updates(), _bad_checksum], ids=["empty_document", "bad_checksum"])
def test_counter_equals_traced_launches_when_nothing_is_exported(launches, blob):
    """no change in the batch, no output block: the change passes and the encoder are not launched"""
    b = loro_b200.import_batch([blob()], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    assert b.counters()["changes"] == 0
    n = launches()
    assert n > 0 and b.timings()["kernel_launches"] == n


def test_counter_equals_traced_launches_tree_documents_with_export(launches):
    blobs = [workloads.make_tree_history(50 + i, n_sites=2, n_base=12, n_ops=40, mixed=bool(i))[0] for i in range(2)]
    b = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    assert b.timings()["tree_ops"] > 0
    n = launches()
    assert b.timings()["kernel_launches"] == n


def test_counter_equals_traced_launches_docset_second_generation(launches):
    """the stored blobs of the first import are copied into the second batch, and its documents copied out again"""
    docs = [OracleDoc(70 + i) for i in range(3)]
    first = []
    for d in docs:
        d.text_insert(d.get_text("t"), 0, "first generation")
        d.commit()
        first.append(d.export_updates())
    vvs = [d.oplog_vv() for d in docs]
    ds = loro_b200.DocSet(lib_path=EMU)
    b1 = ds.import_(first, [1, 2, 3])
    n1 = launches()
    assert b1.timings()["kernel_launches"] == n1
    second = []
    for d, vv in zip(docs, vvs):
        d.text_insert(d.get_text("t"), 5, " second")
        d.commit()
        second.append(d.export_updates(vv))
    b2 = ds.import_(second, [1, 2, 3])
    n2 = launches()
    assert b2.status(0).code == 0 and b2.json_bytes(0) == docs[0].json_text()
    assert n2 > n1 and b2.timings()["kernel_launches"] == n2    # one more launch: the stored blobs copied in
    ds.close()


def test_counter_includes_a_later_export_from_a_version(launches):
    a = OracleDoc(9)
    t = a.get_text("t")
    a.text_insert(t, 0, "hello")
    a.commit()
    vv = a.oplog_vv()
    a.text_insert(t, 5, " world")
    a.commit()
    b = loro_b200.import_batch(mixed_documents() + [a.export_updates()], flags=api.LB_FLAG_EXPORT, lib_path=EMU)
    n = launches()
    assert b.timings()["kernel_launches"] == n
    assert b.export_updates(5, from_vv=vv) == a.export_updates(vv)
    m = launches()
    assert m > 0 and b.timings()["kernel_launches"] == n + m


@pytest.mark.parametrize("n_docs", [0, 1])
def test_phase_times_are_finite_and_not_negative(n_docs):
    blobs = []
    for i in range(n_docs):
        a = OracleDoc(1 + i)
        a.text_insert(a.get_text("t"), 0, "abc")
        blobs.append(a.export_updates())
    tm = loro_b200.import_batch(blobs, lib_path=EMU).timings()
    for k in PHASES:
        assert math.isfinite(tm[k]) and tm[k] >= 0, (k, tm[k])
