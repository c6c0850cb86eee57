"""ctypes binding of include/loro_b200.h (the same stub a cgo/N-API/Rust `extern "C"` shim would bind)."""
import ctypes
import json
import os
from collections import namedtuple

_HERE = os.path.dirname(os.path.abspath(__file__))
_DEFAULT_LIB = os.path.join(_HERE, "libloro_b200.so")

LB_FLAG_NO_JSON = 1
LB_FLAG_KEEP_DEVICE = 2
LB_FLAG_EXPORT = 4
LB_FLAG_COMPACT = 8
LB_FLAG_ATTRIBUTION = 16
LB_FLAG_CURSORS = 32
LB_CURSOR_ID_NOT_FOUND = 100        # CannotFindRelativePosition::IdNotFound
LB_CURSOR_CONTAINER_DELETED = 101   # CannotFindRelativePosition::ContainerDeleted
CONTAINER_TYPES = {"Map": 0, "List": 1, "Text": 2, "Tree": 3, "MovableList": 4, "Counter": 5}

DOC_CODES = {0: "Ok", 1: "DecodeError", 2: "DecodeChecksumMismatchError", 3: "IncompatibleFutureEncodingError",
             4: "DecodeDataCorruptionError", 5: "Unsupported", 6: "CapacityExceeded", 7: "FrontiersNotFound"}

ImportStatus = namedtuple("ImportStatus", "code success pending")


class EngineUnavailable(RuntimeError):
    """The CUDA library is missing or no CUDA device is present (there is no CPU fallback)."""


class DocError(RuntimeError):
    def __init__(self, code):
        super().__init__(DOC_CODES.get(code, str(code)))
        self.code = code


class _Blob(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_char_p), ("len", ctypes.c_size_t), ("doc_id", ctypes.c_uint64)]


class _Options(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int), ("flags", ctypes.c_uint32), ("reserved", ctypes.c_uint32 * 6)]


class _IdSpan(ctypes.Structure):
    _fields_ = [("peer", ctypes.c_uint64), ("start", ctypes.c_int32), ("end", ctypes.c_int32)]


class _Version(ctypes.Structure):
    _fields_ = [("doc_id", ctypes.c_uint64), ("frontiers", ctypes.POINTER(_IdSpan)), ("n_frontiers", ctypes.c_size_t)]


class _ExportRequest(ctypes.Structure):
    _fields_ = [("doc", ctypes.c_size_t), ("from_", ctypes.POINTER(_IdSpan)), ("n_from", ctypes.c_size_t)]


class _RangeRequest(ctypes.Structure):
    _fields_ = [("doc", ctypes.c_size_t), ("spans", ctypes.POINTER(_IdSpan)), ("n_spans", ctypes.c_size_t)]


class _JsonRequest(ctypes.Structure):
    _fields_ = [("doc", ctypes.c_size_t), ("start", ctypes.POINTER(_IdSpan)), ("n_start", ctypes.c_size_t),
                ("end", ctypes.POINTER(_IdSpan)), ("n_end", ctypes.c_size_t), ("flags", ctypes.c_uint32)]


LB_JSON_NO_PEER_COMPRESSION = 1


class _Cursor(ctypes.Structure):
    _fields_ = [("doc", ctypes.c_size_t), ("name", ctypes.c_char_p), ("name_len", ctypes.c_size_t),
                ("peer", ctypes.c_uint64), ("counter", ctypes.c_int32), ("is_root", ctypes.c_uint8),
                ("type", ctypes.c_uint8), ("has_id", ctypes.c_uint8), ("side", ctypes.c_int8),
                ("id_peer", ctypes.c_uint64), ("id_counter", ctypes.c_int32)]


class _CursorResult(ctypes.Structure):
    _fields_ = [("status", ctypes.c_int32), ("side", ctypes.c_int8), ("has_update", ctypes.c_uint8),
                ("update_has_id", ctypes.c_uint8), ("update_side", ctypes.c_int8), ("pos", ctypes.c_uint64),
                ("update_peer", ctypes.c_uint64), ("update_counter", ctypes.c_int32), ("reserved", ctypes.c_uint32),
                ("update_origin_pos", ctypes.c_uint64)]


def parse_container_id(cid):
    """ContainerID's display form ("cid:root-<name>:<Type>" or "cid:<counter>@<peer>:<Type>", as Batch.attribution
    lists containers) -> (is_root, name bytes or None, peer, counter, type code)"""
    if not cid.startswith("cid:") or ":" not in cid[4:]:
        raise ValueError(f"not a container id: {cid!r}")
    body, tname = cid[4:].rsplit(":", 1)
    if tname not in CONTAINER_TYPES:
        raise ValueError(f"unknown container type in {cid!r}")
    if body.startswith("root-"):
        return True, body[5:].encode(), 0, 0, CONTAINER_TYPES[tname]
    counter, peer = body.split("@")
    return False, None, int(peer), int(counter), CONTAINER_TYPES[tname]


class _Status(ctypes.Structure):
    _fields_ = [("code", ctypes.c_int), ("n_success", ctypes.c_size_t), ("success", ctypes.POINTER(_IdSpan)),
                ("n_pending", ctypes.c_size_t), ("pending", ctypes.POINTER(_IdSpan))]


class _Counters(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in ("docs", "docs_ok", "blob_bytes", "blocks", "changes", "op_rows",
                                                "atom_ops", "pending_changes", "json_bytes", "state_hash")]


class _Timings(ctypes.Structure):
    _fields_ = [(n, ctypes.c_float) for n in ("h2d", "frame", "decode", "resolve", "classify", "integrate",
                                               "materialise", "d2h", "total_device", "reexport")] + \
               [("decode_bytes_read", ctypes.c_uint64), ("decode_bytes_written", ctypes.c_uint64),
                ("kernel_launches", ctypes.c_uint32), ("export_bytes", ctypes.c_uint64),
                ("tree", ctypes.c_float), ("reserved0", ctypes.c_uint32), ("tree_ops", ctypes.c_uint64),
                ("decode_fast_blocks", ctypes.c_uint64), ("decode_lane_blocks", ctypes.c_uint64),
                ("decode_unstaged_blocks", ctypes.c_uint64),
                ("alloc_host_ms", ctypes.c_float), ("reserved1", ctypes.c_uint32), ("device_bytes", ctypes.c_uint64),
                ("host_call_ms", ctypes.c_float), ("host_tail_ms", ctypes.c_float), ("attribution", ctypes.c_float),
                ("cursors", ctypes.c_float)]


_libs = {}


def library_path():
    return _DEFAULT_LIB


def load_library(path=None):
    path = path or os.environ.get("LORO_B200_LIB") or _DEFAULT_LIB
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise EngineUnavailable(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). loro_b200 has no CPU fallback.")
    L = ctypes.CDLL(path)
    vp = ctypes.c_void_p
    L.lb_import_batch.argtypes = [ctypes.POINTER(_Blob), ctypes.c_size_t, ctypes.POINTER(_Options), ctypes.POINTER(vp)]
    L.lb_import_batch_device.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32),
                                         ctypes.c_size_t, ctypes.POINTER(_Options), ctypes.POINTER(vp)]
    L.lb_doc_count.restype = ctypes.c_size_t
    L.lb_doc_count.argtypes = [vp]
    L.lb_doc_status.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(_Status)]
    L.lb_doc_json.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t)]
    L.lb_doc_attribution.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t)]
    L.lb_batch_cursor_pos.argtypes = [vp, ctypes.POINTER(_Cursor), ctypes.c_size_t, ctypes.POINTER(_CursorResult)]
    L.lb_doc_export_updates.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(_IdSpan), ctypes.c_size_t,
                                        ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_size_t)]
    L.lb_batch_export_updates.argtypes = [vp, ctypes.POINTER(_ExportRequest), ctypes.c_size_t, ctypes.POINTER(vp)]
    L.lb_batch_export_json_updates.argtypes = [vp, ctypes.POINTER(_JsonRequest), ctypes.c_size_t, ctypes.POINTER(vp)]
    L.lb_batch_export_updates_in_range.argtypes = [vp, ctypes.POINTER(_RangeRequest), ctypes.c_size_t, ctypes.POINTER(vp)]
    L.lb_exports_get.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_size_t)]
    L.lb_exports_free.argtypes = [vp]
    L.lb_doc_vv.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(ctypes.POINTER(_IdSpan)), ctypes.POINTER(ctypes.c_size_t)]
    L.lb_doc_frontiers.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(ctypes.POINTER(_IdSpan)), ctypes.POINTER(ctypes.c_size_t)]
    L.lb_batch_counters.argtypes = [vp, ctypes.POINTER(_Counters)]
    L.lb_batch_timings.argtypes = [vp, ctypes.POINTER(_Timings)]
    L.lb_last_error.restype = ctypes.c_char_p
    L.lb_batch_free.argtypes = [vp]
    L.lb_debug_table.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t),
                                 ctypes.POINTER(ctypes.c_size_t)]
    L.lb_docset_new.argtypes = [ctypes.POINTER(_Options), ctypes.POINTER(vp)]
    L.lb_docset_import.argtypes = [vp, ctypes.POINTER(_Blob), ctypes.c_size_t, ctypes.POINTER(_Options), ctypes.POINTER(vp)]
    L.lb_import_batch_at.argtypes = [ctypes.POINTER(_Blob), ctypes.c_size_t, ctypes.POINTER(_Version), ctypes.c_size_t,
                                     ctypes.POINTER(_Options), ctypes.POINTER(vp)]
    L.lb_docset_checkout.argtypes = [vp, ctypes.POINTER(_Version), ctypes.c_size_t, ctypes.POINTER(_Options),
                                     ctypes.POINTER(vp)]
    L.lb_docset_read.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), ctypes.c_size_t, ctypes.POINTER(_Options),
                                 ctypes.POINTER(vp)]
    L.lb_docset_doc_count.restype = ctypes.c_size_t
    L.lb_docset_doc_count.argtypes = [vp]
    L.lb_docset_stored_bytes.restype = ctypes.c_uint64
    L.lb_docset_stored_bytes.argtypes = [vp]
    L.lb_docset_free.argtypes = [vp]
    _libs[path] = L
    return L


class EngineError(RuntimeError):
    """A C-ABI call returned a non-zero lb_status; .status carries it (6 = LB_ERR_UNSUPPORTED)."""

    def __init__(self, msg, status):
        super().__init__(msg)
        self.status = status


def _check(L, rc, what):
    if rc == 0:
        return
    msg = L.lb_last_error().decode(errors="replace")
    if rc == 2:
        raise EngineUnavailable(f"{what}: {msg}")
    raise EngineError(f"{what} failed (lb_status={rc}): {msg}", rc)


class Batch:
    """Result of one batched import; owns the engine-side outputs until closed."""

    def __init__(self, L, handle, keep=None):
        self._L = L
        self._h = handle
        self._keep = keep  # keeps input buffers alive for device-resident imports
        self.n_docs = L.lb_doc_count(handle)

    def close(self):
        if self._h:
            self._L.lb_batch_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def status(self, i):
        st = _Status()
        _check(self._L, self._L.lb_doc_status(self._h, i, ctypes.byref(st)), "lb_doc_status")
        suc = {st.success[k].peer: (st.success[k].start, st.success[k].end) for k in range(st.n_success)}
        pen = {st.pending[k].peer: (st.pending[k].start, st.pending[k].end) for k in range(st.n_pending)}
        return ImportStatus(st.code, suc, pen or None)

    def export_updates(self, i, from_vv=None):
        """LoroDoc::export(ExportMode::updates(from_vv)) of document i, all_updates when from_vv is None
        (needs flags=LB_FLAG_EXPORT at import).  from_vv: {peer: first counter the receiver lacks}."""
        p = ctypes.c_void_p()
        n = ctypes.c_size_t()
        spans, k = _vv_spans(from_vv)
        _check(self._L, self._L.lb_doc_export_updates(self._h, i, spans, k, ctypes.byref(p), ctypes.byref(n)),
               "lb_doc_export_updates")
        return ctypes.string_at(p.value, n.value)

    def export_updates_many(self, requests):
        """export_updates for many documents in one call (lb_batch_export_updates): `requests` = [(doc, from_vv or
        None), ...].  Returns one entry per request: the bytes, or the EngineError of a request that failed (returned,
        not raised).  A bad document index or a batch without LB_FLAG_EXPORT raises."""
        requests = list(requests)
        arr = (_ExportRequest * max(len(requests), 1))()
        keep = []
        for j, (doc, from_vv) in enumerate(requests):
            spans, k = _vv_spans(from_vv)
            keep.append(spans)
            arr[j].doc = doc
            arr[j].from_ = spans
            arr[j].n_from = k
        h = ctypes.c_void_p()
        _check(self._L, self._L.lb_batch_export_updates(self._h, arr, len(requests), ctypes.byref(h)),
               "lb_batch_export_updates")
        return self._exports(h, len(requests), "export request")

    def export_updates_in_range(self, i, spans):
        """LoroDoc::export(ExportMode::UpdatesInRange { spans }) of document i (needs flags=LB_FLAG_EXPORT at import):
        the changes in `spans` = [(peer, start, end), ...], counters [start, end), taken in the order given."""
        return self._one(self.export_updates_in_range_many([(i, spans)]))

    def export_updates_till(self, i, vv):
        """LoroDoc::export(ExportMode::updates_till(vv)) of document i: one span [0, vv[peer]) per peer
        (encoding.rs:140-151)."""
        return self.export_updates_in_range(i, _till_spans(vv))

    def export_updates_in_range_many(self, requests):
        """export_updates_in_range for many (document, spans) requests in one call (lb_batch_export_updates_in_range).
        Returns one entry per request: the bytes, or the EngineError of a request that failed or was refused (returned,
        not raised).  A bad document index or a batch without LB_FLAG_EXPORT raises."""
        requests = list(requests)
        arr = (_RangeRequest * max(len(requests), 1))()
        keep = []
        for j, (doc, spans) in enumerate(requests):
            spans = list(spans)
            sp = (_IdSpan * max(len(spans), 1))()
            for k, (peer, start, end) in enumerate(spans):
                sp[k].peer, sp[k].start, sp[k].end = int(peer), int(start), int(end)
            keep.append(sp)
            arr[j].doc = doc
            arr[j].spans = sp
            arr[j].n_spans = len(spans)
        h = ctypes.c_void_p()
        _check(self._L, self._L.lb_batch_export_updates_in_range(self._h, arr, len(requests), ctypes.byref(h)),
               "lb_batch_export_updates_in_range")
        return self._exports(h, len(requests), "range request")

    @staticmethod
    def _one(answers):
        """the answer of a one-request *_many call: its value, or its EngineError raised"""
        if isinstance(answers[0], EngineError):
            raise answers[0]
        return answers[0]

    def _exports(self, h, n, what, text=False):
        """the n answers of an lb_exports (freed here): bytes (text: str), or the EngineError of a failed request"""
        out = []
        try:
            for j in range(n):
                p = ctypes.c_void_p()
                ln = ctypes.c_size_t()
                rc = self._L.lb_exports_get(h, j, ctypes.byref(p), ctypes.byref(ln))
                if rc == 0:
                    b = ctypes.string_at(p.value, ln.value)
                    out.append(b.decode("utf-8") if text else b)
                else:
                    msg = self._L.lb_last_error().decode(errors="replace")
                    out.append(EngineError(f"{what} {j} failed (lb_status={rc}): {msg}", rc))
        finally:
            self._L.lb_exports_free(h)
        return out

    def export_json_updates(self, i, start_vv=None, end_vv=None, peer_compression=True):
        """LoroDoc::export_json_updates(start_vv, end_vv) of document i as JSON text (needs flags=LB_FLAG_EXPORT at
        import).  start_vv=None is the empty version; end_vv=None is the document's oplog vv.  Versions are
        {peer: counter}; peer_compression=False gives real peer ids and "peers": null."""
        return self._one(self.export_json_updates_many([(i, start_vv, end_vv, peer_compression)]))

    def export_json_updates_many(self, requests):
        """export_json_updates for many (document, version range) requests in one call (lb_batch_export_json_updates):
        `requests` = [(doc, start_vv, end_vv[, peer_compression]), ...], None versions as in export_json_updates.
        Returns one entry per request: the JSON text, or the EngineError of a request that failed (returned, not raised).
        A bad document index or a batch without LB_FLAG_EXPORT raises."""
        requests = [tuple(r) for r in requests]
        arr = (_JsonRequest * max(len(requests), 1))()
        keep = []
        for j, r in enumerate(requests):
            doc, start_vv, end_vv = r[:3]
            compress = r[3] if len(r) > 3 else True
            if end_vv is None and 0 <= doc < self.n_docs:
                end_vv = self.oplog_vv(doc)
            s_spans, s_n = _vv_spans(start_vv)
            e_spans, e_n = _vv_spans(end_vv)
            keep.append((s_spans, e_spans))
            arr[j].doc = doc
            arr[j].start, arr[j].n_start = s_spans, s_n
            arr[j].end, arr[j].n_end = e_spans, e_n
            arr[j].flags = 0 if compress else LB_JSON_NO_PEER_COMPRESSION
        h = ctypes.c_void_p()
        _check(self._L, self._L.lb_batch_export_json_updates(self._h, arr, len(requests), ctypes.byref(h)),
               "lb_batch_export_json_updates")
        return self._exports(h, len(requests), "json request", text=True)

    def json_bytes(self, i):
        p = ctypes.c_char_p()
        n = ctypes.c_size_t()
        _check(self._L, self._L.lb_doc_json(self._h, i, ctypes.byref(p), ctypes.byref(n)), "lb_doc_json")
        return ctypes.string_at(p, n.value)

    def attribution_bytes(self, i):
        """who wrote document i's state, as the engine's canonical JSON (lb_doc_attribution; needs
        flags=LB_FLAG_ATTRIBUTION at import).  Empty for a document that failed to import."""
        p = ctypes.c_char_p()
        n = ctypes.c_size_t()
        _check(self._L, self._L.lb_doc_attribution(self._h, i, ctypes.byref(p), ctypes.byref(n)), "lb_doc_attribution")
        return ctypes.string_at(p, n.value)

    def attribution(self, i):
        """attribution_bytes(i) parsed, peer indices resolved to peer ids: {container id: entry}, where a Text / List
        entry is [(peer, counter, len), ...] (the ids of its visible elements, in runs), a Map entry {key: (peer,
        lamport, present)} (the winning write of every key, LoroMap::get_last_editor) and a Tree entry {node: (peer,
        counter, alive)} (the node's last move, LoroTree::get_last_move_id).  None for a document that failed."""
        raw = self.attribution_bytes(i)
        if not raw:
            return None
        doc = json.loads(raw)
        peers = [int(p) for p in doc["peers"]]
        out = {}
        for cid, entry in doc["containers"].items():
            if isinstance(entry, list):
                out[cid] = [(peers[p], c, n) for p, c, n in entry]
            else:
                out[cid] = {k: (peers[p], c, bool(f)) for k, (p, c, f) in entry.items()}
        return out

    def cursor_pos(self, cursors):
        """LoroDoc::get_cursor_pos for many cursors in one call (lb_batch_cursor_pos; needs flags=LB_FLAG_CURSORS at
        import).  cursors: [(doc, container, id, side), ...] with container a ContainerID display string
        ("cid:root-text:Text", "cid:3@7:List"), id (peer, counter) or None, side -1 / 0 / 1.  Returns one
        (status, pos, side, update) per cursor: status 0 or LB_CURSOR_* or an lb_status; update None or
        (id or None, side, origin_pos)."""
        cursors = list(cursors)
        n = len(cursors)
        arr = (_Cursor * max(n, 1))()
        keep = []
        for k, (doc, cid, tid, side) in enumerate(cursors):
            is_root, name, peer, counter, ctype = parse_container_id(cid)
            c = arr[k]
            c.doc, c.is_root, c.type, c.side = doc, is_root, ctype, side
            if is_root:
                keep.append(name)
                c.name, c.name_len = name, len(name)
            else:
                c.peer, c.counter = peer, counter
            if tid is not None:
                c.has_id, c.id_peer, c.id_counter = 1, tid[0], tid[1]
        res = (_CursorResult * max(n, 1))()
        _check(self._L, self._L.lb_batch_cursor_pos(self._h, arr, n, res), "lb_batch_cursor_pos")
        out = []
        for r in res[:n]:
            upd = None
            if r.has_update:
                upd = ((r.update_peer, r.update_counter) if r.update_has_id else None, r.update_side, r.update_origin_pos)
            out.append((r.status, r.pos, r.side, upd))
        return out

    def fetch_json(self):
        """make sure the JSON of every document of the batch is in host memory (one download of the whole buffer)"""
        if self.n_docs:
            self.json_bytes(0)

    def fetch_exports(self):
        """same for the re-exported blobs (needs LB_FLAG_EXPORT)"""
        if self.n_docs:
            self.export_updates(0)

    def get_deep_value(self, i):
        st = self.status(i)
        if st.code != 0:
            raise DocError(st.code)
        return json.loads(self.json_bytes(i))

    def oplog_vv(self, i):
        spans = ctypes.POINTER(_IdSpan)()
        n = ctypes.c_size_t()
        _check(self._L, self._L.lb_doc_vv(self._h, i, ctypes.byref(spans), ctypes.byref(n)), "lb_doc_vv")
        return {spans[k].peer: spans[k].end for k in range(n.value)}

    def oplog_frontiers(self, i):
        """LoroDoc::oplog_frontiers(): sorted list of (peer, counter) head ids."""
        spans = ctypes.POINTER(_IdSpan)()
        n = ctypes.c_size_t()
        _check(self._L, self._L.lb_doc_frontiers(self._h, i, ctypes.byref(spans), ctypes.byref(n)), "lb_doc_frontiers")
        return sorted((spans[k].peer, spans[k].start) for k in range(n.value))

    def counters(self):
        c = _Counters()
        _check(self._L, self._L.lb_batch_counters(self._h, ctypes.byref(c)), "lb_batch_counters")
        return {n: getattr(c, n) for n, _ in _Counters._fields_}

    def timings(self):
        t = _Timings()
        _check(self._L, self._L.lb_batch_timings(self._h, ctypes.byref(t)), "lb_batch_timings")
        return {n: getattr(t, n) for n, _ in _Timings._fields_}

    def debug_table(self, name):
        import numpy as np
        n = ctypes.c_size_t()
        es = ctypes.c_size_t()
        _check(self._L, self._L.lb_debug_table(self._h, name.encode(), None, 0, ctypes.byref(n), ctypes.byref(es)),
               "lb_debug_table")
        dt = {1: np.uint8, 2: np.uint16, 4: np.int32, 8: np.int64}[es.value]
        arr = np.empty(n.value, dtype=dt)
        _check(self._L, self._L.lb_debug_table(self._h, name.encode(), arr.ctypes.data, arr.nbytes, ctypes.byref(n),
                                               ctypes.byref(es)), "lb_debug_table")
        return arr


class MultiBatch:
    """A large host batch imported as consecutive sub-batches, two C-ABI calls in flight: while one sub-batch computes,
    the next one's blobs go through the pinned staging ring and the previous one's JSON / exported blobs come home
    (documents are independent, so the split changes no result).  Same accessors as Batch; document i lives in the
    sub-batch that holds it."""

    def __init__(self, parts):
        self._parts = parts
        self._bounds = [0]
        for p in parts:
            self._bounds.append(self._bounds[-1] + p.n_docs)
        self.n_docs = self._bounds[-1]

    def _loc(self, i):
        import bisect
        if not 0 <= i < self.n_docs:
            raise IndexError(i)
        k = bisect.bisect_right(self._bounds, i) - 1
        return self._parts[k], i - self._bounds[k]

    def status(self, i): p, j = self._loc(i); return p.status(j)
    def json_bytes(self, i): p, j = self._loc(i); return p.json_bytes(j)
    def attribution_bytes(self, i): p, j = self._loc(i); return p.attribution_bytes(j)
    def attribution(self, i): p, j = self._loc(i); return p.attribution(j)
    def get_deep_value(self, i): p, j = self._loc(i); return p.get_deep_value(j)
    def oplog_vv(self, i): p, j = self._loc(i); return p.oplog_vv(j)
    def oplog_frontiers(self, i): p, j = self._loc(i); return p.oplog_frontiers(j)
    def export_updates(self, i, from_vv=None): p, j = self._loc(i); return p.export_updates(j, from_vv)

    def _many(self, method, requests):
        """Batch.<method> for requests (doc, ...) with every request sent to its sub-batch: one call per sub-batch, the
        answers in request order"""
        requests = [tuple(r) for r in requests]
        per_part = {}
        for k, r in enumerate(requests):
            p, j = self._loc(r[0])
            per_part.setdefault(id(p), (p, []))[1].append((k, (j,) + r[1:]))
        out = [None] * len(requests)
        for p, reqs in per_part.values():
            for (k, _), res in zip(reqs, getattr(p, method)([r for _, r in reqs])):
                out[k] = res
        return out

    def export_updates_many(self, requests):
        """Batch.export_updates_many with every request sent to its sub-batch: one C call per sub-batch."""
        return self._many("export_updates_many", requests)

    def cursor_pos(self, cursors):
        """Batch.cursor_pos with every cursor sent to its sub-batch: one C call per sub-batch, answers in request order"""
        return self._many("cursor_pos", cursors)

    def export_updates_in_range(self, i, spans): p, j = self._loc(i); return p.export_updates_in_range(j, spans)
    def export_updates_till(self, i, vv): p, j = self._loc(i); return p.export_updates_till(j, vv)

    def export_updates_in_range_many(self, requests):
        """Batch.export_updates_in_range_many with every request sent to its sub-batch: one C call per sub-batch."""
        return self._many("export_updates_in_range_many", requests)

    def export_json_updates(self, i, start_vv=None, end_vv=None, peer_compression=True):
        p, j = self._loc(i)
        return p.export_json_updates(j, start_vv, end_vv, peer_compression)

    def export_json_updates_many(self, requests):
        """Batch.export_json_updates_many with every request sent to its sub-batch: one C call per sub-batch."""
        return self._many("export_json_updates_many", requests)

    def fetch_json(self):
        for p in self._parts:
            p.fetch_json()

    def fetch_exports(self):
        for p in self._parts:
            p.fetch_exports()

    def counters(self):
        out = {}
        for p in self._parts:
            for k, v in p.counters().items():
                out[k] = (out.get(k, 0) ^ v) if k == "state_hash" else out.get(k, 0) + v
        return out

    def timings(self):
        """per-phase device times summed over the sub-batches (they overlap on the device: the sum is not a wall time)"""
        out = {}
        for p in self._parts:
            for k, v in p.timings().items():
                out[k] = out.get(k, 0) + v
        return out

    def close(self):
        for p in self._parts:
            p.close()
        self._parts = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


SPLIT_MIN_BYTES = 256 << 20   # host batches at least this large are imported as overlapping sub-batches ...
SPLIT_MIN_PART_DOCS = 2048    # ... of at least this many documents each (one warp per document: fewer would idle the SMs)
SPLIT_PARTS = 2


def auto_split(blobs):
    """number of sub-batches import_batch uses for `blobs` when the caller does not say"""
    n = len(blobs)
    forced = os.environ.get("LORO_B200_SPLIT")     # measurement hook: force the number of sub-batches
    if forced:
        return max(1, int(forced))
    if n < 2 * SPLIT_MIN_PART_DOCS:
        return 1
    total = 0
    for b in blobs:
        total += len(b)
        if total >= SPLIT_MIN_BYTES:
            return max(1, min(SPLIT_PARTS, n // SPLIT_MIN_PART_DOCS))
    return 1


def _open_batch(L, entry, device, flags, *args, keep=None):
    """Call the C entry point `entry(*args, options, &batch)` and wrap the batch it returns."""
    opt = _Options(device=device, flags=flags)
    h = ctypes.c_void_p()
    _check(L, entry(*args, ctypes.byref(opt), ctypes.byref(h)), entry.__name__)
    return Batch(L, h.value, keep=keep)


def _import_one(L, blobs, device, flags, doc_ids):
    arr, keep = _blob_array(blobs, doc_ids)
    return _open_batch(L, L.lb_import_batch, device, flags, arr, len(blobs))


def import_batch(blobs, device=0, flags=0, lib_path=None, doc_ids=None, split=None):
    """LoroDoc::import for a batch: one fresh document per blob (bytes-like), host buffers in.
    `doc_ids` (one int per blob) groups blobs into documents the way LoroDoc::import_batch takes several updates:
    blobs with the same id form one document; documents are numbered in order of first appearance.
    `split`: number of sub-batches (None = auto_split(blobs) for batches without doc_ids: up to SPLIT_PARTS once the
    batch holds SPLIT_MIN_BYTES, never fewer than SPLIT_MIN_PART_DOCS documents each): sub-batches are imported two
    at a time so that the host<->device transfers of one overlap the kernels of the other; the result is a MultiBatch."""
    L = load_library(lib_path)
    n = len(blobs)
    if split is None:
        split = auto_split(blobs) if doc_ids is None else 1
    if split > 1 and doc_ids is None and n >= 2 * split:
        import threading
        step = (n + split - 1) // split
        ranges = [(a, min(n, a + step)) for a in range(0, n, step)]
        parts = [None] * len(ranges)
        errs = []
        nxt = [0]
        lock = threading.Lock()

        def work():
            while True:
                with lock:
                    k = nxt[0]
                    nxt[0] += 1
                if k >= len(ranges) or errs:
                    return
                a, b = ranges[k]
                try:
                    parts[k] = _import_one(L, blobs[a:b], device, flags, None)
                    if flags & LB_FLAG_EXPORT:
                        parts[k].fetch_exports()    # this sub-batch's blobs come home while the next one computes
                except Exception as e:   # noqa: BLE001 -- re-raised below
                    errs.append(e)

        ts = [threading.Thread(target=work) for _ in range(2)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        if errs:
            for p in parts:
                if p is not None:
                    p.close()
            raise errs[0]
        return MultiBatch(parts)
    return _import_one(L, blobs, device, flags, doc_ids)


def import_batch_at(blobs, versions, doc_ids=None, device=0, flags=0, lib_path=None):
    """import_batch(blobs, doc_ids=doc_ids) followed by LoroDoc::checkout(frontiers) of every document named in
    `versions`: {doc_id: [(peer, counter), ...]} (an empty list is the empty version).  Documents not named stay at the
    latest version.  A frontier id the document does not hold gives that document code 7 (FrontiersNotFound)."""
    L = load_library(lib_path)
    arr, keep = _blob_array(blobs, doc_ids)
    ver, vkeep = _version_array(list(versions.items()))
    return _open_batch(L, L.lb_import_batch_at, device, flags, arr, len(blobs), ver, len(versions))


def _till_spans(vv):
    """ExportMode::updates_till(vv) as spans (encoding.rs:140-151): [0, vv[peer]) for every peer of vv"""
    return [(p, 0, c) for p, c in dict(vv or {}).items()]


def _vv_spans(from_vv):
    """{peer: counter} -> (lb_id_span array or None, count) in the form lb_doc_export_updates takes"""
    if not from_vv:
        return None, 0
    spans = (_IdSpan * len(from_vv))()
    for j, (peer, ctr) in enumerate(from_vv.items()):
        spans[j].peer = peer
        spans[j].start = 0
        spans[j].end = ctr
    return spans, len(from_vv)


def _version_array(requests):
    """[(doc_id, [(peer, counter), ...]), ...] -> lb_version array (+ the span arrays it points into)"""
    arr = (_Version * max(len(requests), 1))()
    keep = []
    for i, (doc_id, frontiers) in enumerate(requests):
        frontiers = list(frontiers)
        spans = (_IdSpan * max(len(frontiers), 1))()
        for k, (peer, ctr) in enumerate(frontiers):
            spans[k].peer = int(peer)
            spans[k].start = int(ctr)
            spans[k].end = int(ctr) + 1
        keep.append(spans)
        arr[i].doc_id = int(doc_id)
        arr[i].frontiers = spans
        arr[i].n_frontiers = len(frontiers)
    return arr, keep


def _blob_array(blobs, doc_ids):
    n = len(blobs)
    arr = (_Blob * max(n, 1))()
    keep = []
    for i, b in enumerate(blobs):
        b = bytes(b)
        keep.append(b)
        arr[i].ptr = b
        arr[i].len = len(b)
        arr[i].doc_id = i if doc_ids is None else int(doc_ids[i])
    return arr, keep


class DocSet:
    """Persistent documents: LoroDoc::import / import_batch against documents that already hold history.  The documents
    live in device memory between calls (their change stores in wire form, include/loro_b200.h lb_docset_*); every
    import_() returns a Batch that answers for the documents it touched -- status of THIS import, state after it."""

    def __init__(self, device=0, lib_path=None):
        self._L = load_library(lib_path)
        self._device = device
        opt = _Options(device=device, flags=0)
        h = ctypes.c_void_p()
        _check(self._L, self._L.lb_docset_new(ctypes.byref(opt), ctypes.byref(h)), "lb_docset_new")
        self._h = h.value

    def import_(self, blobs, doc_ids, flags=0):
        """blobs[i] is imported into document doc_ids[i]; several blobs for one id = import_batch on that document.
        Documents of the returned Batch are numbered in order of first appearance of their id."""
        arr, keep = _blob_array(blobs, doc_ids)
        return _open_batch(self._L, self._L.lb_docset_import, self._device, flags, self._h, arr, len(blobs))

    def checkout(self, requests, flags=0):
        """The stored documents at earlier versions: `requests` = [(doc_id, [(peer, counter), ...]), ...].  Document i of
        the returned Batch is request i (a doc_id may repeat; one the set has never seen is an empty document).  The set is
        not modified."""
        requests = list(requests)
        ver, keep = _version_array(requests)
        return _open_batch(self._L, self._L.lb_docset_checkout, self._device, flags, self._h, ver, len(requests))

    def read(self, doc_ids, flags=0):
        """The stored documents as they are, nothing imported (lb_docset_read): document i of the returned Batch is
        doc_ids[i] (an id the set has never seen is an empty document), imported with LB_FLAG_EXPORT so that
        export_updates / export_updates_many answer for it.  The set is not modified."""
        doc_ids = [int(d) for d in doc_ids]
        ids = (ctypes.c_uint64 * max(len(doc_ids), 1))(*doc_ids)
        return _open_batch(self._L, self._L.lb_docset_read, self._device, flags, self._h, ids, len(doc_ids))

    @property
    def n_docs(self):
        return self._L.lb_docset_doc_count(self._h)

    @property
    def stored_bytes(self):
        return self._L.lb_docset_stored_bytes(self._h)

    def close(self):
        if self._h:
            self._L.lb_docset_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def import_batch_device(d_bytes_ptr, offsets, lens, device=0, flags=0, lib_path=None, keep=None):
    """Same with blobs already resident in HBM: `d_bytes_ptr` is a device pointer (int); blob i occupies
    [offsets[i], offsets[i] + lens[i]) with every offset a multiple of 16."""
    L = load_library(lib_path)
    n = len(offsets)
    assert len(lens) == n
    if hasattr(offsets, "ctypes"):  # numpy fast path
        import numpy as np
        o = np.ascontiguousarray(offsets, dtype=np.uint64)
        l_ = np.ascontiguousarray(lens, dtype=np.uint32)
        offs = o.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))
        ls = l_.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))
        keep = (keep, o, l_)
    else:
        offs = (ctypes.c_uint64 * max(n, 1))(*[int(x) for x in offsets])
        ls = (ctypes.c_uint32 * max(n, 1))(*[int(x) for x in lens])
    return _open_batch(L, L.lb_import_batch_device, device, flags, ctypes.c_void_p(d_bytes_ptr), offs, ls, n, keep=keep)


def device_trim(device=0, lib_path=None):
    """Release the device blocks the engine keeps for the next batch (lb_device_trim)."""
    L = load_library(lib_path)
    _check(L, L.lb_device_trim(int(device)), "lb_device_trim")


def numa_bind(device=0, lib_path=None):
    """Pin this process (its current thread and the threads created from it) to the CPUs of the NUMA node of `device`.
    Returns True when the binding was applied."""
    L = load_library(lib_path)
    L.lb_numa_bind.argtypes = [ctypes.c_int]
    return L.lb_numa_bind(device) == 0


def pack_blobs(blobs):
    """Concatenate blobs at 16-byte aligned starts -> (bytes, offsets, lens) for import_batch_device."""
    import numpy as np
    lens = np.fromiter((len(b) for b in blobs), dtype=np.uint32, count=len(blobs))
    padded = (lens.astype(np.uint64) + 15) & ~np.uint64(15)
    offs = np.zeros(len(blobs), dtype=np.uint64)
    if len(blobs):
        offs[1:] = np.cumsum(padded)[:-1]
    total = int(padded.sum())
    buf = np.zeros(total + 64, dtype=np.uint8)
    for b, o in zip(blobs, offs):
        buf[int(o):int(o) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return buf, offs, lens
