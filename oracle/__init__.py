"""ORACLE (test infrastructure) -- ctypes wrapper over oracle/liboracle.so.

A CPU restatement of the reference's import/merge/export path (see oracle/doc.hpp for the
file:line map).  It is the *checker*: only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this package.  The product (loro_b200/) never does.
"""
import ctypes
import json
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

CT_MAP, CT_LIST, CT_TEXT, CT_TREE, CT_MOVABLE, CT_COUNTER = 0, 1, 2, 3, 4, 5


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("capi.cpp", "doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
    if not force and os.path.exists(_LIB_PATH):
        try:
            if all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
                return _LIB_PATH
        except OSError:
            return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s", "liboracle.so"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        vp, sz, u8p = ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint8)
        L.lo_doc_new.restype = vp
        L.lo_doc_new.argtypes = [ctypes.c_uint64]
        L.lo_doc_free.argtypes = [vp]
        L.lo_set_peer.argtypes = [vp, ctypes.c_uint64]
        L.lo_free.argtypes = [vp]
        L.lo_get_container.argtypes = [vp, ctypes.c_char_p, sz, ctypes.c_int]
        L.lo_text_insert.argtypes = [vp, ctypes.c_int, sz, ctypes.c_char_p, sz]
        L.lo_list_insert.argtypes = [vp, ctypes.c_int, sz, sz, ctypes.POINTER(ctypes.c_int),
                                     ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_double),
                                     ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(sz)]
        L.lo_seq_delete.argtypes = [vp, ctypes.c_int, sz, sz]
        L.lo_list_insert_tagged.argtypes = [vp, ctypes.c_int, sz, sz, ctypes.c_char_p]
        L.lo_map_set_tagged.argtypes = [vp, ctypes.c_int, ctypes.c_char_p, sz, ctypes.c_char_p]
        L.lo_seq_len.argtypes = [vp, ctypes.c_int]
        L.lo_map_set.argtypes = [vp, ctypes.c_int, ctypes.c_char_p, sz, ctypes.c_int, ctypes.c_int64,
                                 ctypes.c_double, ctypes.c_char_p, sz]
        L.lo_map_delete.argtypes = [vp, ctypes.c_int, ctypes.c_char_p, sz]
        L.lo_child_container.argtypes = [vp, ctypes.c_uint64, ctypes.c_int, ctypes.c_int]
        L.lo_next_counter.argtypes = [vp]
        L.lo_tree_create.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, ctypes.c_int,
                                     ctypes.POINTER(ctypes.c_int)]
        L.lo_tree_move.argtypes = [vp, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, ctypes.c_int, ctypes.c_uint64,
                                   ctypes.c_int, ctypes.c_int]
        L.lo_tree_delete.argtypes = [vp, ctypes.c_int, ctypes.c_uint64, ctypes.c_int]
        L.lo_tree_meta.argtypes = [vp, ctypes.c_uint64, ctypes.c_int]
        L.lo_tree_nodes.argtypes = [vp, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int),
                                    ctypes.c_int]
        L.lo_commit.argtypes = [vp]
        L.lo_export.argtypes = [vp, sz, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int32),
                                ctypes.POINTER(vp), ctypes.POINTER(sz)]
        L.lo_import.argtypes = [vp, ctypes.c_char_p, sz, ctypes.POINTER(vp)]
        L.lo_json.restype = vp
        L.lo_json.argtypes = [vp, ctypes.POINTER(sz)]
        L.lo_vv_json.restype = vp
        L.lo_vv_json.argtypes = [vp]
        L.lo_frontiers_json.restype = vp
        L.lo_frontiers_json.argtypes = [vp]
        L.lo_pending_count.argtypes = [vp]
        L.lo_inconsistent_delete.argtypes = [vp]
        L.lo_len_ops.restype = ctypes.c_int64
        L.lo_len_ops.argtypes = [vp]
        L.lo_decode_dump.restype = vp
        L.lo_decode_dump.argtypes = [ctypes.c_char_p, sz, ctypes.c_int, ctypes.POINTER(sz)]
        L.lo_block_roundtrip.argtypes = [ctypes.c_char_p, sz, ctypes.c_int, ctypes.POINTER(vp), ctypes.POINTER(sz)]
        L.lo_codec.argtypes = [ctypes.c_char_p, ctypes.c_char_p, sz, ctypes.c_int64, ctypes.POINTER(vp),
                               ctypes.POINTER(sz)]
        L.lo_bench_import.restype = ctypes.c_int64
        L.lo_bench_import.argtypes = [ctypes.c_void_p, ctypes.c_void_p, sz, ctypes.c_int, ctypes.c_int,
                                      ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_double)]
        _lib = L
    return _lib


def _take_str(ptr, n=None):
    L = lib()
    s = ctypes.string_at(ptr, n) if n is not None else ctypes.string_at(ptr)
    L.lo_free(ptr)
    return s


def _take_bytes(ptr, n):
    b = ctypes.string_at(ptr, n)
    lib().lo_free(ptr)
    return b


class ImportError_(Exception):
    def __init__(self, code, msg=""):
        super().__init__(f"import failed code={code} {msg}")
        self.code = code


def _uleb(b, i):
    v, sh = 0, 0
    while True:
        c = b[i]
        i += 1
        v |= (c & 0x7f) << sh
        sh += 7
        if not c & 0x80:
            return v, i


def blob_mode(blob):
    """encode mode of a blob (u16 big endian at [20..22), encoding.rs:299-330); 0xFFFF when too short"""
    return (blob[20] << 8) | blob[21] if len(blob) >= 22 else 0xFFFF


def blob_change_num(blob):
    """ImportBlobMetadata.change_num of a FastUpdates blob: the sum of the blocks' n_changes (the fifth varint of
    every EncodedBlock envelope, block_encode.rs:95-119)"""
    total, i, n = 0, 22, len(blob)
    try:
        while i < n:
            ln, i = _uleb(blob, i)
            end, j, x = i + ln, i, 0
            for _ in range(5):
                x, j = _uleb(blob, j)
            total += x
            i = end
    except IndexError:
        pass
    return total


class OracleDoc:
    """Mirrors the slice of LoroDoc the hot path needs (crates/loro/src/lib.rs:425-866,1235)."""

    def __init__(self, peer=0):
        self._d = lib().lo_doc_new(peer)
        self.peer = peer

    def __del__(self):
        try:
            if self._d:
                lib().lo_doc_free(self._d)
                self._d = None
        except Exception:
            pass

    def set_peer_id(self, peer):
        lib().lo_set_peer(self._d, peer)
        self.peer = peer

    def container(self, name, ctype):
        b = name.encode()
        return lib().lo_get_container(self._d, b, len(b), ctype)

    def get_text(self, name): return self.container(name, CT_TEXT)
    def get_list(self, name): return self.container(name, CT_LIST)
    def get_map(self, name): return self.container(name, CT_MAP)
    def get_tree(self, name): return self.container(name, CT_TREE)

    # ---- movable tree (handler/tree.rs): nodes are (peer, counter) TreeIDs, parent None = root
    def tree_create(self, c, parent=None, index=-1):
        out = ctypes.c_int()
        pp, pc = parent if parent else (0, 0)
        if lib().lo_tree_create(self._d, c, 0 if parent else 1, pp, pc, index, ctypes.byref(out)) != 0:
            raise IndexError("tree_create rejected")
        return (self.peer, out.value)

    def tree_move(self, c, target, parent=None, index=-1):
        pp, pc = parent if parent else (0, 0)
        if lib().lo_tree_move(self._d, c, target[0], target[1], 0 if parent else 1, pp, pc, index) != 0:
            raise IndexError("tree_move rejected (cycle, dead node or index out of range)")

    def tree_delete(self, c, target):
        if lib().lo_tree_delete(self._d, c, target[0], target[1]) != 0:
            raise IndexError("tree_delete rejected")

    def tree_meta(self, target):
        return lib().lo_tree_meta(self._d, target[0], target[1])

    def tree_nodes(self, c):
        n = lib().lo_tree_nodes(self._d, c, None, None, 0)
        peers = (ctypes.c_uint64 * max(n, 1))()
        ctrs = (ctypes.c_int * max(n, 1))()
        lib().lo_tree_nodes(self._d, c, peers, ctrs, n)
        return [(int(peers[i]), int(ctrs[i])) for i in range(n)]

    def text_insert(self, c, pos, s):
        b = s.encode()
        if lib().lo_text_insert(self._d, c, pos, b, len(b)) != 0:
            raise IndexError("text_insert out of range")

    def _vals(self, values):
        n = len(values)
        kinds = (ctypes.c_int * n)()
        ints = (ctypes.c_int64 * n)()
        f64s = (ctypes.c_double * n)()
        strs = (ctypes.c_char_p * n)()
        slens = (ctypes.c_size_t * n)()
        for i, v in enumerate(values):
            if v is None: kinds[i] = 0
            elif v is True: kinds[i] = 1
            elif v is False: kinds[i] = 2
            elif isinstance(v, int): kinds[i] = 3; ints[i] = v
            elif isinstance(v, float): kinds[i] = 4; f64s[i] = v
            elif isinstance(v, str):
                b = v.encode(); kinds[i] = 5; strs[i] = b; slens[i] = len(b)
            elif isinstance(v, bytes): kinds[i] = 6; strs[i] = v; slens[i] = len(v)
            elif isinstance(v, tuple) and v[0] == "container": kinds[i] = 9; ints[i] = v[1]
            else: raise TypeError(v)
        return n, kinds, ints, f64s, strs, slens

    @staticmethod
    def _tagged(v):
        import struct
        if v is None: return b"\x00"
        if v is True: return b"\x01"
        if v is False: return b"\x02"
        if isinstance(v, int): return b"\x03" + struct.pack("<q", v)
        if isinstance(v, float): return b"\x04" + struct.pack("<d", v)
        if isinstance(v, str):
            b = v.encode()
            return b"\x05" + struct.pack("<I", len(b)) + b
        if isinstance(v, bytes): return b"\x06" + struct.pack("<I", len(v)) + v
        if isinstance(v, (list, tuple)): return b"\x07" + struct.pack("<I", len(v)) + b"".join(OracleDoc._tagged(x) for x in v)
        if isinstance(v, dict):
            out = b"\x08" + struct.pack("<I", len(v))
            for k, x in v.items():
                kb = k.encode()
                out += struct.pack("<I", len(kb)) + kb + OracleDoc._tagged(x)
            return out
        raise TypeError(v)

    @staticmethod
    def _nested(values):
        return any(isinstance(v, (list, dict)) for v in values)

    def list_insert(self, c, pos, *values):
        if self._nested(values):   # LoroValue::List / Map items (encoding/value.rs:1027-1036)
            if lib().lo_list_insert_tagged(self._d, c, pos, len(values), b"".join(self._tagged(v) for v in values)) != 0:
                raise IndexError("list_insert out of range")
            return
        n, kinds, ints, f64s, strs, slens = self._vals(values)
        if lib().lo_list_insert(self._d, c, pos, n, kinds, ints, f64s, strs, slens) != 0:
            raise IndexError("list_insert out of range")

    def list_insert_container(self, c, pos, ctype):
        ctr = lib().lo_next_counter(self._d)
        self.list_insert(c, pos, ("container", ctype))
        return lib().lo_child_container(self._d, self.peer, ctr, ctype)

    def delete(self, c, pos, length):
        if lib().lo_seq_delete(self._d, c, pos, length) != 0:
            raise IndexError("delete out of range")

    def seq_len(self, c):
        return lib().lo_seq_len(self._d, c)

    def map_set(self, c, key, v):
        k = key.encode()
        if self._nested([v]):
            lib().lo_map_set_tagged(self._d, c, k, len(k), self._tagged(v))
            return
        n, kinds, ints, f64s, strs, slens = self._vals([v])
        # the payload itself: reading strs[0] back returns the bytes cut at the first NUL, slens[0] does not
        payload = v.encode() if isinstance(v, str) else v if isinstance(v, bytes) else b""
        lib().lo_map_set(self._d, c, k, len(k), kinds[0], ints[0], f64s[0], payload, slens[0])

    def map_set_container(self, c, key, ctype):
        ctr = lib().lo_next_counter(self._d)
        self.map_set(c, key, ("container", ctype))
        return lib().lo_child_container(self._d, self.peer, ctr, ctype)

    def map_delete(self, c, key):
        k = key.encode()
        lib().lo_map_delete(self._d, c, k, len(k))

    def commit(self):
        lib().lo_commit(self._d)

    def export_updates(self, from_vv=None):
        from_vv = from_vv or {}
        n = len(from_vv)
        peers = (ctypes.c_uint64 * max(n, 1))(*[int(p) for p in from_vv.keys()])
        ctrs = (ctypes.c_int32 * max(n, 1))(*[int(c) for c in from_vv.values()])
        out = ctypes.c_void_p()
        ln = ctypes.c_size_t()
        rc = lib().lo_export(self._d, n, peers, ctrs, ctypes.byref(out), ctypes.byref(ln))
        if rc != 0:
            raise RuntimeError("export failed")
        return _take_bytes(out.value, ln.value)

    def import_(self, blob):
        st = ctypes.c_void_p()
        rc = lib().lo_import(self._d, blob, len(blob), ctypes.byref(st))
        status = json.loads(_take_str(st.value))
        if rc != 0:
            raise ImportError_(rc, status.get("err", ""))
        return {
            "success": {int(k): tuple(v) for k, v in status["success"].items()},
            "pending": {int(k): tuple(v) for k, v in status["pending"].items()} or None,
        }

    def import_batch(self, blobs):
        """LoroDoc::import_batch (loro.rs:1183-1290): the blobs are imported one after the other, sorted by
        (mode, number of changes descending) (stable), and the statuses folded -- success keeps the start of the first
        blob that reported the peer and the highest end, pending keeps the lowest start and the LOWEST end."""
        if not blobs:
            return {"success": {}, "pending": None}
        if len(blobs) == 1:
            return self.import_(blobs[0])
        order = sorted(range(len(blobs)), key=lambda i: (blob_mode(blobs[i]), -blob_change_num(blobs[i])))
        success, pending, err = {}, {}, None
        for i in order:
            try:
                st = self.import_(blobs[i])
            except ImportError_ as e:
                err = e
                continue
            for peer, (a, b) in st["success"].items():
                success[peer] = (success[peer][0], max(success[peer][1], b)) if peer in success else (a, b)
            for peer, (a, b) in (st["pending"] or {}).items():
                pending[peer] = (min(pending[peer][0], a), min(pending[peer][1], b)) if peer in pending else (a, b)
        if err:
            raise err
        return {"success": success, "pending": pending or None}

    def json_text(self):
        ln = ctypes.c_size_t()
        p = lib().lo_json(self._d, ctypes.byref(ln))
        return _take_str(p, ln.value)

    def get_deep_value(self):
        t = self.json_text()
        if t.startswith(b"!error"):
            raise RuntimeError(t.decode())
        return json.loads(t)

    def oplog_vv(self):
        return {int(k): v for k, v in json.loads(_take_str(lib().lo_vv_json(self._d))).items()}

    def frontiers(self):
        return [(int(p), c) for p, c in json.loads(_take_str(lib().lo_frontiers_json(self._d)))]

    def pending_count(self): return lib().lo_pending_count(self._d)
    def inconsistent_delete(self): return bool(lib().lo_inconsistent_delete(self._d))
    def len_ops(self): return lib().lo_len_ops(self._d)


def decode_dump(blob, raw_block=False):
    ln = ctypes.c_size_t()
    p = lib().lo_decode_dump(blob, len(blob), 1 if raw_block else 0, ctypes.byref(ln))
    return json.loads(_take_str(p, ln.value))


def block_roundtrip(block, section=-1):
    out = ctypes.c_void_p()
    ln = ctypes.c_size_t()
    rc = lib().lo_block_roundtrip(block, len(block), section, ctypes.byref(out), ctypes.byref(ln))
    b = _take_bytes(out.value, ln.value)
    if rc != 0:
        raise RuntimeError(b.decode(errors="replace"))
    return b


def codec(op, data=b"", arg=0):
    """Codec primitive hook. i64 arrays travel as little-endian 8-byte values."""
    out = ctypes.c_void_p()
    ln = ctypes.c_size_t()
    rc = lib().lo_codec(op.encode(), data, len(data), arg, ctypes.byref(out), ctypes.byref(ln))
    b = _take_bytes(out.value, ln.value)
    if rc != 0:
        raise ValueError(f"{op}: {b.decode(errors='replace')}")
    return b


def i64s(b):
    import struct
    return list(struct.unpack("<%dq" % (len(b) // 8), b))


def pack_i64s(vals):
    import struct
    return struct.pack("<%dq" % len(vals), *vals)


def _bench_worker(args):
    buf, offs, want_json, want_export = args
    import numpy as np
    return _bench_import_threads(np.frombuffer(buf, dtype=np.uint8), offs, 1, want_json, want_export)


def _bench_import_threads(buf, offsets, threads, want_json, want_export):
    import numpy as np
    offs = np.ascontiguousarray(np.asarray(offsets, dtype=np.uint64))
    h = ctypes.c_uint64()
    secs = ctypes.c_double()
    flags = (1 if want_json else 0) | (2 if want_export else 0)
    ops = lib().lo_bench_import(buf.ctypes.data, offs.ctypes.data, len(offs) - 1, threads, flags,
                                ctypes.byref(h), ctypes.byref(secs))
    return {"ops": ops, "seconds": secs.value, "hash": h.value}


def bench_import(blob_concat, offsets, threads=1, want_json=True, want_export=False, processes=False):
    """CPU-baseline leg: import each doc into a fresh oracle doc on `threads` host cores.
    With processes=True the docs are split over `threads` single-threaded worker processes (one doc per task
    inside each), which scales far better than threads sharing one malloc arena set."""
    import time
    import numpy as np
    buf = np.frombuffer(blob_concat, dtype=np.uint8) if not isinstance(blob_concat, np.ndarray) else blob_concat
    n = len(offsets) - 1
    if not processes or threads <= 1 or n < 2 * threads:
        return _bench_import_threads(buf, offsets, threads, want_json, want_export)
    import multiprocessing as mp
    per = (n + threads - 1) // threads
    tasks = []
    for w in range(threads):
        lo, hi = w * per, min(n, (w + 1) * per)
        if lo >= hi:
            break
        base = int(offsets[lo])
        tasks.append((buf[base:int(offsets[hi])].tobytes(), [int(o) - base for o in offsets[lo:hi + 1]], want_json, want_export))
    ctx = mp.get_context("fork")
    with ctx.Pool(len(tasks)) as pool:
        pool.map(_noop, range(len(tasks)))          # spin the workers up outside the timed region
        t0 = time.time()
        rs = pool.map(_bench_worker, tasks)
        dt = time.time() - t0
    h = 0
    for r in rs:
        h ^= r["hash"]
    return {"ops": sum(r["ops"] for r in rs), "seconds": dt, "hash": h}


def _noop(_):
    return 0
