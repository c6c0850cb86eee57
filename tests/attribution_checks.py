"""Shared checks for attribution (lb_doc_attribution): the engine's bytes of a document against the oracle-side reference
(tests/attribution_ref.cpp), at the latest version or at requested Frontiers."""
import ctypes
import hashlib
import json
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_ref = None


def _ref_lib():
    """tests/attribution_ref.cpp built once per source version into the temporary directory (the tree may be read-only)"""
    global _ref
    if _ref is None:
        srcs = [os.path.join(HERE, "attribution_ref.cpp")] + [os.path.join(ROOT, "oracle", f) for f in
                                                               ("doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
        h = hashlib.sha256()
        for s in srcs:
            with open(s, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "loro_b200_attribution_ref_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.at_attribution.restype = ctypes.c_void_p
        L.at_attribution.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64),
                                     ctypes.POINTER(ctypes.c_int32), ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.at_free.argtypes = [ctypes.c_void_p]
        _ref = L
    return _ref


def attribution_at(doc, frontiers=None):
    """The reference attribution of an OracleDoc as bytes: at the latest version (frontiers None) or at `frontiers`
    [(peer, counter), ...]; None when the frontiers are not in its DAG."""
    L = _ref_lib()
    at = frontiers is not None
    frontiers = list(frontiers or [])
    n = len(frontiers)
    peers = (ctypes.c_uint64 * max(n, 1))(*[int(p) for p, _ in frontiers])
    ctrs = (ctypes.c_int32 * max(n, 1))(*[int(c) for _, c in frontiers])
    ln = ctypes.c_size_t()
    p = L.at_attribution(doc._d, 1 if at else 0, peers, ctrs, n, ctypes.byref(ln))
    out = ctypes.string_at(p, ln.value)
    L.at_free(p)
    if out == b"!FrontiersNotFound":
        return None
    assert not out.startswith(b"!error"), out
    return out


def parsed(raw):
    """attribution bytes -> (peers as ints, containers dict), as Batch.attribution resolves them"""
    d = json.loads(raw)
    return [int(p) for p in d["peers"]], d["containers"]
