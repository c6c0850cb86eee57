"""Shared checks for LoroDoc::export_json_updates (json_schema.rs): the oracle-side reference (tests/json_updates_ref.cpp,
built on the unchanged oracle), the invariants every export satisfies, and the engine-against-reference comparison."""
import ctypes
import hashlib
import json
import os
import random
import subprocess
import tempfile

from oracle import OracleDoc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_ref = None


def _ref_lib():
    """tests/json_updates_ref.cpp built once per source version into the temporary directory (the tree may be read-only)"""
    global _ref
    if _ref is None:
        srcs = [os.path.join(HERE, "json_updates_ref.cpp")] + [os.path.join(ROOT, "oracle", f) for f in
                                                                ("doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
        h = hashlib.sha256()
        for s in srcs:
            with open(s, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "loro_b200_json_ref_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        vvp = [ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int32), ctypes.c_size_t]
        L.jx_export.restype = ctypes.c_void_p
        L.jx_export.argtypes = [ctypes.c_void_p] + vvp + vvp + [ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]
        L.jx_commit_with.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int]
        L.jx_free.argtypes = [ctypes.c_void_p]
        _ref = L
    return _ref


def _vv_args(vv):
    vv = dict(vv or {})
    n = len(vv)
    peers = (ctypes.c_uint64 * max(n, 1))(*[int(p) for p in vv])
    ctrs = (ctypes.c_int32 * max(n, 1))(*[int(c) for c in vv.values()])
    return peers, ctrs, n


def export_json_updates(doc, start_vv=None, end_vv=None, peer_compression=True):
    """The reference's JSON text for oracle document `doc`; end_vv=None is its oplog vv."""
    L = _ref_lib()
    if end_vv is None:
        end_vv = doc.oplog_vv()
    ln = ctypes.c_size_t()
    p = L.jx_export(doc._d, *_vv_args(start_vv), *_vv_args(end_vv), int(bool(peer_compression)), ctypes.byref(ln))
    out = ctypes.string_at(p, ln.value)
    L.jx_free(p)
    assert not out.startswith(b"!error"), out
    return out.decode("utf-8")


def commit_with(doc, timestamp, msg=None):
    """commit the oracle document's open transaction with a timestamp and an optional commit message"""
    m = (msg or "").encode()
    _ref_lib().jx_commit_with(doc._d, int(timestamp), m, len(m), int(msg is not None))


def oracle_doc(blobs):
    d = OracleDoc(1)
    d.import_batch(list(blobs))
    return d


def _parse_id(s, peers):
    c, p = s.split("@")
    p = int(p)
    return (peers[p] if peers is not None else p), int(c)


def op_len(op):
    c = op["content"]
    if c["type"] == "insert":
        if "text" in c:
            return len(c["text"])
        if "pos" in c:
            return len(c["value"])
        return 1
    if c["type"] == "delete" and "len" in c:
        return abs(c["len"])
    return 1


def _register_order(ch):
    """the peer indices of one change in encode_change's register order (json_schema.rs:301-548): per op its container
    (normal ids), the containers among its values, a delete's start id, a tree op's target and parent; then the change id;
    then its deps"""
    out = []

    def cid_peer(c):
        if c.startswith("🦜:"):
            c = c[len("🦜:"):]
        if c.startswith("cid:") and not c.startswith("cid:root-"):
            out.append(int(c.split(":")[1].split("@")[1]))
    for o in ch["ops"]:
        cid_peer(o["container"])
        c = o["content"]
        vals = c.get("value", []) if "pos" in c else ([c["value"]] if "value" in c else [])
        for v in vals:
            if isinstance(v, str):
                cid_peer(v)
        for k in ("start_id", "target", "parent"):
            if isinstance(c.get(k), str):
                out.append(int(c[k].split("@")[1]))
    out.append(int(ch["id"].split("@")[1]))
    out += [int(d.split("@")[1]) for d in ch["deps"]]
    return out


def check_invariants(text, start_vv, end_vv, oplog_vv):
    """What every export between two versions satisfies: per peer the change ids cover exactly [start, end) (after
    refine_vv), each change's op lengths add up to its atom count and its ops are contiguous, lamports never decrease,
    and with peer compression the peers are indexed in order of first use."""
    j = json.loads(text)
    assert list(j) == ["schema_version", "start_version", "peers", "changes"]
    peers = [int(p) for p in j["peers"]] if j["peers"] is not None else None

    def refine(vv):
        return {p: min(c, oplog_vv.get(p, 0)) for p, c in (vv or {}).items() if c > 0 and oplog_vv.get(p, 0) > 0}
    s, e = refine(start_vv), refine(end_vv)
    covered = {}
    last_lamport = -1
    used = []
    for ch in j["changes"]:
        assert list(ch) == ["id", "timestamp", "deps", "lamport", "msg", "ops"]
        if peers is not None:
            used += _register_order(ch)
        peer, c0 = _parse_id(ch["id"], peers)
        n = 0
        for o in ch["ops"]:
            assert list(o) == ["container", "content", "counter"]
            assert o["counter"] == c0 + n, (o, c0, n)
            n += op_len(o)
        assert n > 0
        covered.setdefault(peer, []).append((c0, c0 + n))
        assert ch["lamport"] >= last_lamport
        last_lamport = ch["lamport"]
    for p, spans in covered.items():
        spans.sort()
        assert spans[0][0] == s.get(p, 0), (p, spans[0], s.get(p, 0))
        assert spans[-1][1] == e.get(p, 0), (p, spans[-1], e.get(p, 0))
        for a, b in zip(spans, spans[1:]):
            assert a[1] == b[0]
    for p in set(e) | set(s):
        if e.get(p, 0) > s.get(p, 0):
            assert p in covered, p
    if peers is not None:
        # peer indices are handed out in order of first use: the first uses read 0, 1, 2, ...
        seen = []
        for x in used:
            if x not in seen:
                seen.append(x)
        assert seen == list(range(len(peers))), seen
    return j


def random_range(rng, vv):
    """a random (start, end) pair over `vv`: cuts inside changes and ops, and now and then end <= start, an empty end, an
    unknown peer or a counter past the vv"""
    peers = list(vv)

    def pick():
        v = {}
        for p in peers:
            r = rng.random()
            if r < 0.15:
                continue
            v[p] = vv[p] + rng.randint(1, 5) if r > 0.9 else rng.randint(0, vv[p])
        if rng.random() < 0.1:
            v[0xFEEDFACE] = rng.randint(1, 9)
        return v
    a, b = pick(), pick()
    k = rng.random()
    if k < 0.1:
        return b, {}
    if k < 0.55:
        return {p: min(a.get(p, 0), b.get(p, 0)) for p in set(a) | set(b)}, {p: max(a.get(p, 0), b.get(p, 0)) for p in set(a) | set(b)}
    return a, b


def compare_batch(batch, oracles, ranges, peer_compression=(True, False)):
    """Every (doc, start, end) of `ranges`, under each compression setting, in ONE engine call: byte for byte equal to the
    reference on the oracle document, and satisfying the invariants.  Returns the engine texts."""
    reqs = [(d, s, e, pc) for pc in peer_compression for d, s, e in ranges]
    got = batch.export_json_updates_many(reqs)
    for (d, s, e, pc), g in zip(reqs, got):
        assert isinstance(g, str), (d, s, e, pc, g)
        want = export_json_updates(oracles[d], s, e, pc)
        assert g == want, "doc %d start %r end %r compression %r\nengine %s\noracle %s" % (d, s, e, pc, g[:600], want[:600])
        check_invariants(g, s, oracles[d].oplog_vv() if e is None else e, oracles[d].oplog_vv())
    return got


def seeded_ranges(seed, n_docs, vvs, per_doc=3):
    rng = random.Random(seed)
    out = []
    for d in range(n_docs):
        out.append((d, None, None))
        for _ in range(per_doc):
            s, e = random_range(rng, vvs[d])
            out.append((d, s, e))
    return out
