"""Shared checks for cursors (lb_batch_cursor_pos): the oracle-side reference (tests/cursor_ref.cpp) answering the same
requests as Batch.cursor_pos, in the same form."""
import ctypes
import hashlib
import os
import random
import subprocess
import tempfile

from loro_b200.api import parse_container_id

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_ref = None


def _ref_lib():
    """tests/cursor_ref.cpp built once per source version into the temporary directory (the tree may be read-only)"""
    global _ref
    if _ref is None:
        srcs = [os.path.join(HERE, "cursor_ref.cpp")] + [os.path.join(ROOT, "oracle", f) for f in
                                                         ("doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
        h = hashlib.sha256()
        for s in srcs:
            with open(s, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "loro_b200_cursor_ref_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.cr_open.restype = ctypes.c_void_p
        L.cr_open.argtypes = [ctypes.c_void_p]
        L.cr_close.argtypes = [ctypes.c_void_p]
        L.cr_query.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64,
                               ctypes.c_int32, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_int32, ctypes.c_int,
                               ctypes.POINTER(ctypes.c_int64)]
        _ref = L
    return _ref


def cursor_pos_ref(doc, cursors):
    """The reference's answers for cursors [(container, id | None, side), ...] on an OracleDoc, in Batch.cursor_pos's
    form (status, pos, side, update)"""
    L = _ref_lib()
    cx = L.cr_open(doc._d)
    assert cx
    out = (ctypes.c_int64 * 9)()
    res = []
    try:
        for cid, tid, side in cursors:
            is_root, name, peer, counter, ctype = parse_container_id(cid)
            name = name or b""
            tp, tc = tid if tid is not None else (0, 0)
            L.cr_query(cx, int(is_root), name, len(name), peer, counter, ctype, int(tid is not None), tp, tc, side, out)
            upd = None
            if out[3]:
                upd = ((out[5] & 0xFFFFFFFFFFFFFFFF, out[6]) if out[4] else None, out[7], out[8])
            res.append((out[0], out[1], out[2], upd))
    finally:
        L.cr_close(cx)
    return res


def seq_containers(doc):
    """the Text / List containers of an OracleDoc's attribution, with the ids of their visible elements in order"""
    import json
    from .attribution_checks import attribution_at
    raw = json.loads(attribution_at(doc))
    peers = [int(p) for p in raw["peers"]]
    out = {}
    for cid, entry in raw["containers"].items():
        if cid.endswith(":Text") or cid.endswith(":List"):
            out[cid] = [(peers[p], c + k) for p, c, n in entry for k in range(n)]
    return out


def sample_cursors(rnd, containers, vv, k):
    """k random cursors [(container, id | None, side)] over the given containers: ids drawn from the whole oplog (so
    visible and deleted elements of the container, elements of other containers, ids of delete and map ops), some past
    the oplog vv or of a peer the document lacks, some without an id"""
    cids = sorted(containers)
    peers = sorted(p for p, n in vv.items() if n > 0) or [1]
    out = []
    for _ in range(k):
        cid = rnd.choice(cids)
        p = rnd.choice(peers)
        r = rnd.random()
        if r < 0.85:
            tid = (p, rnd.randrange(max(vv.get(p, 1), 1)))
        elif r < 0.9:
            tid = (p, vv.get(p, 0) + rnd.randint(0, 3))
        elif r < 0.93:
            tid = (p ^ 0x5A5A, 0)
        else:
            tid = None
        out.append((cid, tid, rnd.choice((-1, 0, 1))))
    return out
