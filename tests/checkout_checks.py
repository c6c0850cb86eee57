"""Shared checks for checkout (LoroDoc::checkout(&frontiers) + get_deep_value, loro.rs:1353-1433): the engine's state of a
document at requested Frontiers against the oracle's capped replay (tests/checkout_ref.cpp), JSON byte for byte."""
import ctypes
import hashlib
import os
import random
import subprocess
import tempfile

import oracle
from oracle import OracleDoc

import loro_b200

from . import workloads

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FRONTIERS_NOT_FOUND = 7
_ref = None


def _ref_lib():
    """tests/checkout_ref.cpp built once per source version into the temporary directory (the tree may be read-only)"""
    global _ref
    if _ref is None:
        srcs = [os.path.join(HERE, "checkout_ref.cpp")] + [os.path.join(ROOT, "oracle", f) for f in
                                                            ("doc.hpp", "block.hpp", "codec.hpp", "model.hpp")]
        h = hashlib.sha256()
        for s in srcs:
            with open(s, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "loro_b200_checkout_ref_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.ck_json_at.restype = ctypes.c_void_p
        L.ck_json_at.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int32),
                                 ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.ck_free.argtypes = [ctypes.c_void_p]
        _ref = L
    return _ref


def json_at(doc, frontiers):
    """The oracle document's get_deep_value() at `frontiers` [(peer, counter), ...] as JSON bytes; None when the
    frontiers are not in its DAG (LoroError::FrontiersNotFound)."""
    L = _ref_lib()
    n = len(frontiers)
    peers = (ctypes.c_uint64 * max(n, 1))(*[int(p) for p, _ in frontiers])
    ctrs = (ctypes.c_int32 * max(n, 1))(*[int(c) for _, c in frontiers])
    ln = ctypes.c_size_t()
    p = L.ck_json_at(doc._d, peers, ctrs, n, ctypes.byref(ln))
    out = ctypes.string_at(p, ln.value)
    L.ck_free(p)
    if out == b"!FrontiersNotFound":
        return None
    assert not out.startswith(b"!error"), out
    return out


def oracle_doc(blobs):
    """an oracle document after import_batch(blobs)"""
    d = OracleDoc(1)
    d.import_batch(list(blobs))
    return d


def applied_ids(doc):
    """every applied id of the document, as (peer, counter)"""
    return [(p, c) for p, n in sorted(doc.oplog_vv().items()) for c in range(n)]


def random_frontiers(rnd, doc, max_ids=3):
    """a random Frontiers of the document: 0..max_ids applied ids, sometimes redundant (one in the past of another)"""
    ids = applied_ids(doc)
    if not ids:
        return []
    k = rnd.randint(1, max_ids)
    return [rnd.choice(ids) for _ in range(k)]


def interesting_ids(doc_blob):
    """ids inside changes and inside ops of the blob: the middle of every multi-atom op (text / list inserts, forward and
    reversed delete spans) and of every multi-op change"""
    out = []
    for bl in oracle.decode_dump(doc_blob)["blocks"]:
        for ch in bl["changes"]:
            peer = int(ch["peer"])
            ops = ch["ops"]
            if ops:
                end = ops[-1]["counter"] + ops[-1]["len"]
                if end - ch["counter"] > 1:
                    out.append((peer, ch["counter"] + (end - ch["counter"]) // 2))
            for op in ops:
                if op["len"] > 1:
                    out.append((peer, op["counter"] + op["len"] // 2))
    return out


def check_import_batch_at(groups, requests, lib_path=None, expect_codes=None):
    """groups: the blob lists of the documents (document i = doc_id i); requests: {doc_id: frontiers}.  Every requested
    document must read like the oracle at its frontiers (or fail with FrontiersNotFound exactly when the oracle does), every
    other document like the plain import; vv / frontiers are the oplog's."""
    blobs, ids = [], []
    for i, g in enumerate(groups):
        blobs += list(g)
        ids += [i] * len(g)
    batch = loro_b200.import_batch_at(blobs, requests, doc_ids=ids, lib_path=lib_path)
    plain = loro_b200.import_batch(blobs, doc_ids=ids, lib_path=lib_path)
    assert batch.n_docs == len(groups)
    for i, g in enumerate(groups):
        o = oracle_doc(g)
        st, pst = batch.status(i), plain.status(i)
        assert st.success == pst.success and st.pending == pst.pending, i
        assert batch.oplog_vv(i) == plain.oplog_vv(i) == o.oplog_vv(), i
        assert batch.oplog_frontiers(i) == plain.oplog_frontiers(i), i
        if i not in requests:
            assert st.code == pst.code, i
            assert pst.code != 0 or batch.json_bytes(i) == plain.json_bytes(i), i
            continue
        want = json_at(o, requests[i])
        if expect_codes and i in expect_codes:
            assert st.code == expect_codes[i], (i, st.code)
        if want is None:
            assert st.code == FRONTIERS_NOT_FOUND, (i, st.code, requests[i])
            continue
        if pst.code != 0:                       # unsupported ops: decided over the whole history
            assert st.code == pst.code, (i, st.code, pst.code)
            continue
        assert st.code == 0, (i, st.code, requests[i])
        got = batch.json_bytes(i)
        assert got == want, (i, requests[i], got[:400], want[:400])
    return batch


def history_snapshots(seed, n_sites=3, n_ops=200, tree=False):
    """A make_doc_history-style run that, every few steps, commits a site and records that site's own JSON and frontiers
    (the second formulation of "the state at F": what the site saw).  Returns (blob of the synced document, snapshots)."""
    rnd = random.Random(seed)
    peers = [rnd.getrandbits(64) | 1 for _ in range(n_sites)]
    docs = [OracleDoc(p) for p in peers]
    hs = [(d.get_text("text"), d.get_list("list"), d.get_map("map")) for d in docs]
    trees = [d.get_tree("tree") for d in docs] if tree else None
    snaps = []
    for step in range(n_ops):
        i = rnd.randrange(n_sites)
        if tree and rnd.random() < 0.5:
            workloads.random_tree_edit(rnd, docs[i], trees[i])
        else:
            workloads.random_edit(rnd, docs[i], *hs[i])
        if rnd.random() < 0.3:
            docs[i].commit()
        if rnd.random() < 0.08:
            j = rnd.randrange(n_sites)
            if j != i:
                workloads.merge(docs[j], docs[i])
        if rnd.random() < 0.15:
            k = rnd.randrange(n_sites)
            docs[k].commit()
            snaps.append((docs[k].frontiers(), docs[k].json_text()))
    for _ in range(2):
        for i in range(n_sites):
            for j in range(n_sites):
                if i != j:
                    workloads.merge(docs[i], docs[j])
    return docs[0].export_updates(), snaps
