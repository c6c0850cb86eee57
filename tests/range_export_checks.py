"""Shared checks for ExportMode::UpdatesInRange (change_store.rs:179-199): the oracle-side reference
(tests/range_export_ref.cpp, built on the unchanged oracle), span sets that exercise its rules, and the
engine-against-reference comparison."""
import ctypes
import hashlib
import os
import random
import subprocess
import tempfile

from oracle import OracleDoc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LACKING_PEER = 0xFEEDFACE
_ref = None


class Refused(Exception):
    """the reference panics on the span set, or would store a change twice"""


def _ref_lib():
    """tests/range_export_ref.cpp built once per source version into the temporary directory (the tree may be read-only)"""
    global _ref
    if _ref is None:
        srcs = [os.path.join(HERE, "range_export_ref.cpp")] + [os.path.join(ROOT, "oracle", f) for f in
                                                                ("doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
        h = hashlib.sha256()
        for s in srcs:
            with open(s, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "loro_b200_range_ref_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.rx_export.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int32),
                                ctypes.POINTER(ctypes.c_int32), ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p),
                                ctypes.POINTER(ctypes.c_size_t)]
        L.rx_free.argtypes = [ctypes.c_void_p]
        _ref = L
    return _ref


def export_in_range(doc, spans):
    """the reference's export(UpdatesInRange { spans }) of oracle document `doc`; spans = [(peer, start, end), ...].
    Raises Refused where the reference panics or would store a change twice."""
    L = _ref_lib()
    n = len(spans)
    peers = (ctypes.c_uint64 * max(n, 1))(*[int(s[0]) for s in spans])
    starts = (ctypes.c_int32 * max(n, 1))(*[int(s[1]) for s in spans])
    ends = (ctypes.c_int32 * max(n, 1))(*[int(s[2]) for s in spans])
    out, ln = ctypes.c_void_p(), ctypes.c_size_t()
    rc = L.rx_export(doc._d, peers, starts, ends, n, ctypes.byref(out), ctypes.byref(ln))
    data = ctypes.string_at(out.value, ln.value)
    L.rx_free(out)
    if rc != 0:
        raise Refused(data.decode())
    return data


def hello_docs():
    """doc_1 and doc_2 of loro_import_batch_status (crates/loro/tests/loro_rust_test.rs:2411-2460)"""
    out = []
    for peer in (1, 2):
        d = OracleDoc(peer)
        d.text_insert(d.get_text("text"), 0, "Hello world!")
        d.commit()
        out.append(d)
    return out


BATCH_STATUS_SPANS = ([(1, 0, 5)], [(1, 5, 7)], [(1, 6, 12)], [(2, 0, 5)], [(2, 5, 6)], [(2, 6, 12)])


def till_spans(vv):
    """ExportMode::updates_till(vv) (encoding.rs:140-151)"""
    return [(p, 0, c) for p, c in vv.items()]


def span_sets(vv, rnd):
    """span sets that exercise the rules: one- and two-sided ranges, several disjoint spans of a peer in shuffled
    order, adjacent spans in both orders, reversed and negative spans, spans past the vv, a lacking peer, nothing"""
    peers = sorted(vv)
    out = [till_spans(vv), [], [(LACKING_PEER, 0, 5)], [(p, c, c + 9) for p, c in vv.items()]]
    out.append([(p, 0, rnd.randint(0, c)) for p, c in vv.items()])                       # updates_till(random vv)
    out.append([(p, rnd.randint(0, c), c) for p, c in vv.items()])                       # updates(from)
    for _ in range(3):                                                                   # two-sided
        s = []
        for p, c in vv.items():
            a = rnd.randint(0, c)
            s.append((p, a, rnd.randint(a, c + 2)))
        out.append(s)
    for p in peers:
        c = vv[p]
        if c < 6:
            continue
        a, b = sorted(rnd.sample(range(1, c), 2))
        out.append([(p, b, c), (p, 0, a)])                  # disjoint, the higher first
        out.append([(p, a, c), (p, 0, a)])                  # adjacent, the higher first: two blocks
        out.append([(p, 0, a), (p, a, c)])                  # adjacent, in order: continues the block
        out.append([(p, 0, a), (p, a, b), (p, b, c + 4)])   # a chain, past the vv
        out.append([(p, b, a)])                             # reversed: covers a+1 .. b+1
        out.append([(p, -3, a)])                            # starts below 0: selects nothing
        out.append([(p, a, -2)])                            # reversed with a negative end: -1 .. a+1
        out.append([(p, b, c), (p, a, b), (p, 0, a)])       # from the top down: three blocks
        out.append([(p, 0, a), (p, b, c)])                  # a gap above an earlier span: refused
        out.append([(p, 0, b), (p, a, c)])                  # overlap: refused
        out.append([(p, a, b), (p, a, b)])                  # the same span twice: refused
        others = [(q, 0, vv[q]) for q in peers if q != p]
        mixed = others + [(p, b, c), (p, 0, a)]
        rnd.shuffle(mixed)
        out.append(mixed)
    return out


def check_requests(batch, refs, reqs, single=True):
    """every answer of one many-request call equals the reference's (refusals: LB_ERR_INVALID_ARG), and, with `single`,
    what a call with that request alone answers"""
    from loro_b200 import api
    got = batch.export_updates_in_range_many(reqs)
    for k, ((i, spans), g) in enumerate(zip(reqs, got)):
        try:
            want = export_in_range(refs[i], spans)
        except Refused:
            assert isinstance(g, api.EngineError) and g.status == 1, (k, i, spans, g)
            continue
        assert g == want, (k, i, spans, g if isinstance(g, Exception) else len(g), len(want))
        if single:
            assert batch.export_updates_in_range(i, spans) == want, (k, i, spans)
    return got


def random_requests(refs, seed, per_doc=None):
    rnd = random.Random(seed)
    reqs = []
    for i, ref in enumerate(refs):
        sets = span_sets(ref.oplog_vv(), rnd)
        if per_doc:
            sets = rnd.sample(sets, min(per_doc, len(sets)))
        reqs += [(i, s) for s in sets]
    reqs += rnd.sample(reqs, min(8, len(reqs)))   # repeats
    rnd.shuffle(reqs)
    return reqs
