"""Phase 7's per-change row pass (a warp per change, 32 rows at a time) against the oracle's export, on change shapes
that sit on its 32-row chunk boundaries: row counts around multiples of 32, text runs placed behind a chosen number of
map rows, delete chains, trimmed changes and changes over the block size.  Shared by test_export_change_rows_emu.py and
test_export_change_rows_gpu.py: every builder returns the blobs of one batch, checked with check_export_against_oracle.

A document's own export holds its ops already merged, so rows of one change that merge only on import come from
blobs that hold the same changes with their ops cut into pieces (tests/change_rows_ref.cpp): there the export's merge
inside a change decides every row, across the 32-row chunks, for single-element deletes in both directions and for
text runs that a string-arena doubling of the importer breaks."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

from oracle import OracleDoc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_ref = None

CHUNK_ROW_COUNTS = [31, 32, 33, 64, 65]
TEXT_RUN_LEADS = [0, 1, 29, 30, 31, 32, 33, 62, 63, 64]
TEXT_RUN_PADS = [20, 30, 40]
DELETE_CHAIN_LENGTHS = [31, 32, 33, 64, 65]
MERGE_DELETE_LENGTHS = [31, 32, 33, 64, 65, 70]
MERGE_DELETE_LEADS = [0, 1, 30, 31, 32, 33]
MERGE_RUN_LEADS = [0, 1, 20, 31, 32, 33, 63]
MERGE_RUN_PADS = [0, 20, 30]
PIECE_SEEDS = [1, 2, 3]


def _ref_lib():
    """tests/change_rows_ref.cpp built once per source version into the temporary directory (the tree may be read-only)"""
    global _ref
    if _ref is None:
        srcs = [os.path.join(HERE, "change_rows_ref.cpp")] + [os.path.join(ROOT, "oracle", f) for f in
                                                              ("doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
        h = hashlib.sha256()
        for src in srcs:
            with open(src, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "loro_b200_change_rows_ref_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.cr_export_pieces.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p),
                                       ctypes.POINTER(ctypes.c_size_t)]
        L.cr_free.argtypes = [ctypes.c_void_p]
        _ref = L
    return _ref


def export_in_pieces(doc, piece=1):
    """doc's all_updates blob with every List / Text insert and delete span cut into ops of `piece` atoms; it must
    be longer than the merged export, or there is nothing for an importer to merge back"""
    L = _ref_lib()
    out, ln = ctypes.c_void_p(), ctypes.c_size_t()
    rc = L.cr_export_pieces(doc._d, piece, ctypes.byref(out), ctypes.byref(ln))
    data = ctypes.string_at(out.value, ln.value)
    L.cr_free(out)
    assert rc == 0, data.decode()
    assert len(data) > len(doc.export_updates())
    return data


def _typing_change(pad, lead, run, seed_text=0):
    """Peer 1 types `run` characters one at a time into a text after `lead` map rows, all in one change, on top of
    `pad` characters it imported from peer 2."""
    a = OracleDoc(2)
    if pad:
        ta = a.get_text("t")
        a.text_insert(ta, 0, "p" * pad)
        a.commit()
    b = OracleDoc(1)
    if pad:
        b.import_(a.export_updates())
    m = b.get_map("m")
    for i in range(lead):
        b.map_set(m, f"k{i}", i)
    t = b.get_text("t")
    for i in range(run):
        b.text_insert(t, pad + i, chr(ord("a") + (seed_text + i) % 26))
    b.commit()
    return b.export_updates()


def chunk_sized_row_counts(n_rows):
    """one change of exactly n_rows rows that never merge (map sets and single list inserts at the front), with and
    without a text run behind them"""
    d = OracleDoc(5)
    m, l = d.get_map("m"), d.get_list("l")
    for i in range(n_rows):
        if i % 3 == 2:
            d.list_insert(l, 0, i)
        else:
            d.map_set(m, f"k{i}", i)
    d.commit()
    blobs = [d.export_updates()]
    e = OracleDoc(6)
    t, l2 = e.get_text("t"), e.get_list("l")
    for i in range(n_rows):
        if i % 2:
            e.text_insert(t, 0, "xy")
        else:
            e.list_insert(l2, 0, i, i + 1)
    e.commit()
    blobs.append(e.export_updates())
    return blobs


def text_runs_on_chunk_boundaries(pad, lead):
    """a typing run over another peer's text whose rows start around rows 31/32 and 63/64 of the change, and whose
    string-arena offsets cross a capacity doubling of the buffer"""
    return [_typing_change(pad, lead, 70)]


def string_generation_runs():
    """runs long enough to cross several doublings of the importer's buffer (32, 64, 128, 256 bytes)"""
    return [_typing_change(pad, lead, run, seed_text=pad)
            for pad, lead, run in [(5, 3, 300), (33, 31, 200), (64, 32, 260), (1, 0, 129)]]


def delete_chains(n):
    """backspace chains (reversed spans), forward-delete chains, and lone deletes next to each other, n deletes per
    change: runs of delete rows in a change of n rows"""
    blobs = []
    for mode in range(3):
        d = OracleDoc(10 + mode)
        l = d.get_list("l")
        d.list_insert(l, 0, *range(4 * n + 8))
        d.commit()
        t = d.get_text("t")
        d.text_insert(t, 0, "z" * (4 * n + 8))
        d.commit()
        for i in range(n):
            if mode == 0:
                d.delete(l, 2 * n - i, 1)            # backspace: one reversed span
            elif mode == 1:
                d.delete(l, 3, 1)                    # forward delete: one span
            else:
                if i % 2:
                    d.delete(l, (5 * i) % (2 * n), 1)   # deletes that do not line up, between text deletes
                else:
                    d.delete(t, (3 * i) % n, 1)
        d.commit()
        blobs.append(d.export_updates())
    return blobs


def check_trimmed_changes(lib_path=None):
    """updates that start inside changes the document already holds: the first kept row of the change is cut"""
    from .docset_checks import check_docset_against_oracle
    check_docset_against_oracle(lib_path=lib_path, n_docs=4, seed=7, rounds=6, edits=40, stale_inside=True)


def change_over_the_block_size():
    """one change whose estimate exceeds MAX_BLOCK_SIZE (split into segments), next to one just under it"""
    blobs = []
    for count in (900, 1100):
        d = OracleDoc(30)
        l = d.get_list("l")
        for i in range(count):
            d.list_insert(l, 0, i)    # single-value rows that never merge: 4 bytes of estimate each
        d.commit()
        blobs.append(d.export_updates())
    d = OracleDoc(31)
    t = d.get_text("t")
    d.text_insert(t, 0, "q" * 5000)   # one text op over the block size: cut by Op::slice
    d.commit()
    blobs.append(d.export_updates())
    return blobs


# ---- rows of one change that merge only on import


def _lead(d, lead):
    m = d.get_map("m")
    for i in range(lead):
        d.map_set(m, f"k{i}", i)


def deletes_merge_into_directed_spans(n, lead):
    """backspace and forward-delete chains of n single-element rows in one change, after `lead` map rows: the
    delete runs straddle rows 31/32 and 63/64, and the first two rows of a run fix its direction"""
    blobs = []
    for mode in range(4):
        d = OracleDoc(40 + mode)
        seq = d.get_text("t") if mode >= 2 else d.get_list("l")
        if mode >= 2:
            d.text_insert(seq, 0, "".join(chr(ord("a") + i % 26) for i in range(2 * n + 8)))
        else:
            d.list_insert(seq, 0, *range(2 * n + 8))
        d.commit()
        _lead(d, lead)
        for i in range(n):
            d.delete(seq, (n + 4 - i) if mode % 2 == 0 else 4, 1)   # backspace: reversed span / forward delete
        d.commit()
        blobs.append(export_in_pieces(d))
    return blobs


def delete_runs_of_several_spans():
    """a change whose delete rows form several runs, of pieces of 1 and 2 elements: a backspace run, a lone delete, a
    forward run, in list and text, each run ending where the next starts to differ"""
    blobs = []
    for piece in (1, 2):
        d = OracleDoc(50 + piece)
        l, t = d.get_list("l"), d.get_text("t")
        d.list_insert(l, 0, *range(200))
        d.text_insert(t, 0, "x" * 200)
        d.commit()
        for i in range(40):
            d.delete(l, 150 - i, 1)
        d.delete(l, 20, 1)
        for i in range(37):
            d.delete(l, 30, 1)
        for i in range(33):
            d.delete(t, 100 - i, 1)
        for i in range(29):
            d.delete(t, 10, 1)
        d.commit()
        blobs.append(export_in_pieces(d, piece))
    return blobs


def text_and_list_runs_across_chunks(pad, lead):
    """typing runs of single-character rows and list runs of single-value rows after `lead` map rows: runs across
    rows 31/32 and 63/64, and text runs that the importer's string-arena doublings (32, 64, 128 bytes) break"""
    d = OracleDoc(60)
    t, l = d.get_text("t"), d.get_list("l")
    if pad:
        d.text_insert(t, 0, "p" * pad)
        d.commit()
    _lead(d, lead)
    for i in range(100):
        d.text_insert(t, pad + i, "é" if i % 7 == 3 else chr(ord("a") + i % 26))
    d.commit()
    _lead(d, lead)
    for i in range(90):
        d.list_insert(l, i, i)
    d.commit()
    return [export_in_pieces(d, 1), export_in_pieces(d, 3)]


def random_histories_in_pieces(seed):
    """multi-site histories with their ops cut into pieces of 1 and 2 atoms"""
    from . import workloads
    blobs = []
    for i in range(3):
        blob = workloads.make_doc_history(seed * 10 + i, n_sites=2 + i, n_ops=200)[0]
        d = OracleDoc(0xABC)
        d.import_(blob)
        blobs.append(export_in_pieces(d, 1 + i % 2))
    return blobs


def change_over_the_block_size_in_pieces():
    """a change over MAX_BLOCK_SIZE whose rows merge back on import before it is split into segments"""
    d = OracleDoc(70)
    t, l = d.get_text("t"), d.get_list("l")
    d.text_insert(t, 0, "q" * 5000)
    d.list_insert(l, 0, *range(1100))
    d.commit()
    return [export_in_pieces(d, 1)]
