"""Known-answer semantics tests restated from the reference's own integration tests.

  crates/loro-internal/tests/fugue.rs:5-90          forward/backward interleaving, Yjs anomaly => "b12"
  crates/loro-internal/tests/test.rs:423-449        pending changes => "0" then "210"
  crates/loro-internal/tests/test.rs:1253-1287      exact ImportStatus ranges
  README.md:75-120                                   two-doc sync example
  crates/loro/tests/issue.rs:257-264                 duplicate import is a no-op
"""
import os
import random

import pytest

import oracle
from oracle import OracleDoc


def merge(a, b):
    """a.merge(&b) == a.import(b.export(updates(a.vv)))"""
    return a.import_(b.export_updates(a.oplog_vv()))


def test_forward_interleaving():
    a, b = OracleDoc(0), OracleDoc(1)
    a.text_insert(a.get_text("text"), 0, "Hello")
    b.text_insert(b.get_text("text"), 0, " World!")
    merge(a, b)
    assert a.get_deep_value() == {"text": "Hello World!"}


def test_backward_interleaving():
    a, b = OracleDoc(0), OracleDoc(1)
    ta, tb = a.get_text("text"), b.get_text("text")
    for ch in "olleH":
        a.text_insert(ta, 0, ch)
    for ch in "!dlroW ":
        b.text_insert(tb, 0, ch)
    assert a.get_deep_value() == {"text": "Hello"}
    merge(a, b)
    assert a.get_deep_value() == {"text": "Hello World!"}


def test_forward_backward():
    a, b = OracleDoc(0), OracleDoc(1)
    ta, tb = a.get_text("text"), b.get_text("text")
    a.text_insert(ta, 0, "ll")
    a.text_insert(ta, 0, "He")
    a.text_insert(ta, 4, "o")
    b.text_insert(tb, 0, " !")
    b.text_insert(tb, 1, "W")
    b.text_insert(tb, 2, "d")
    b.text_insert(tb, 2, "l")
    b.text_insert(tb, 2, "r")
    b.text_insert(tb, 2, "o")
    merge(a, b)
    assert a.get_deep_value() == {"text": "Hello World!"}


def test_yjs_interleave():
    a, b, c = OracleDoc(0), OracleDoc(1), OracleDoc(2)
    c.text_insert(c.get_text("text"), 0, "2")
    merge(a, c)
    a.text_insert(a.get_text("text"), 0, "1")
    b.text_insert(b.get_text("text"), 0, "b")
    merge(a, b)
    assert a.get_deep_value() == {"text": "b12"}
    # and symmetric convergence
    merge(b, a)
    assert b.get_deep_value() == {"text": "b12"}


def test_pending():
    a = OracleDoc(0)
    a.text_insert(a.get_text("text"), 0, "0")
    b = OracleDoc(1)
    b.import_(a.export_updates())
    b.text_insert(b.get_text("text"), 0, "1")
    c = OracleDoc(2)
    c.import_(b.export_updates())
    c.text_insert(c.get_text("text"), 0, "2")
    a.import_(c.export_updates(b.oplog_vv()))
    assert a.get_deep_value() == {"text": "0"}
    assert a.pending_count() == 1
    a.import_(b.export_updates(a.oplog_vv()))
    assert a.get_deep_value() == {"text": "210"}
    assert a.pending_count() == 0


def test_import_status():
    doc = OracleDoc(0)
    doc.text_insert(doc.get_text("text"), 0, "a")
    doc2 = OracleDoc(1)
    t2 = doc2.get_text("text")
    doc2.text_insert(t2, 0, "b")
    doc2.commit()
    update1 = doc2.export_updates()   # the reference test uses a snapshot here; same op content
    vv1 = doc2.oplog_vv()
    doc2.text_insert(t2, 1, "c")
    update2 = doc2.export_updates(vv1)
    s1 = doc.import_(update2)
    s2 = doc.import_(update1)
    assert s1 == {"success": {}, "pending": {1: (1, 2)}}
    assert s2 == {"success": {1: (0, 2)}, "pending": None}
    assert doc.get_deep_value()["text"] in ("abc", "bca")


def test_readme_sync_example():
    a, b = OracleDoc(1), OracleDoc(2)
    la, lb = a.get_list("list"), b.get_list("list")
    a.list_insert(la, 0, "A")
    a.list_insert(la, 1, "B")
    a.list_insert(la, 2, "C")
    b.import_(a.export_updates())
    assert b.get_deep_value() == {"list": ["A", "B", "C"]}
    b.delete(lb, 1, 1)
    a.import_(b.export_updates(a.oplog_vv()))
    assert a.get_deep_value() == {"list": ["A", "C"]} == b.get_deep_value()


def test_import_twice_is_noop():
    a, b = OracleDoc(1), OracleDoc(2)
    a.text_insert(a.get_text("t"), 0, "hello")
    a.map_set(a.get_map("m"), "k", 5)
    blob = a.export_updates()
    s1 = b.import_(blob)
    v1 = b.get_deep_value()
    s2 = b.import_(blob)
    assert s1["success"] == {1: (0, 6)} and s2 == {"success": {}, "pending": None}
    assert b.get_deep_value() == v1 == {"t": "hello", "m": {"k": 5}}
    assert b.export_updates() == blob


def test_map_lww_and_delete():
    a, b = OracleDoc(1), OracleDoc(2)
    ma, mb = a.get_map("m"), b.get_map("m")
    a.map_set(ma, "x", 1)
    b.map_set(mb, "x", 2)     # same lamport, larger peer wins
    b.map_set(mb, "y", "s")
    merge(a, b); merge(b, a)
    assert a.get_deep_value() == b.get_deep_value() == {"m": {"x": 2, "y": "s"}}
    a.map_delete(ma, "y")
    merge(b, a)
    assert b.get_deep_value() == {"m": {"x": 2}}


def test_nested_containers_deep_value():
    a = OracleDoc(7)
    m = a.get_map("root")
    child = a.map_set_container(m, "todo", oracle.CT_LIST)
    a.list_insert(child, 0, 1, "two", None, True, 2.5)
    t = a.list_insert_container(child, 5, oracle.CT_TEXT)
    a.text_insert(t, 0, "hé\"llo\n")
    b = OracleDoc(8)
    b.import_(a.export_updates())
    expect = {"root": {"todo": [1, "two", None, True, 2.5, "hé\"llo\n"]}}
    assert a.get_deep_value() == expect == b.get_deep_value()


def test_unicode_positions():
    a, b = OracleDoc(1), OracleDoc(2)
    ta = a.get_text("t")
    a.text_insert(ta, 0, "añ😀b")
    a.text_insert(ta, 2, "中")
    a.delete(ta, 3, 1)   # the emoji
    b.import_(a.export_updates())
    assert b.get_deep_value() == {"t": "añ中b"}
    b.text_insert(b.get_text("t"), 4, "é")
    merge(a, b)
    assert a.get_deep_value() == {"t": "añ中bé"}


def _random_edit(rnd, d, text, lst, mp):
    r = rnd.random()
    if r < 0.35:
        n = d.seq_len(text)
        d.text_insert(text, rnd.randint(0, n), "".join(rnd.choice("abcdefg xyzé") for _ in range(rnd.randint(1, 4))))
    elif r < 0.5:
        n = d.seq_len(text)
        if n:
            p = rnd.randrange(n)
            d.delete(text, p, min(rnd.randint(1, 3), n - p))
    elif r < 0.75:
        n = d.seq_len(lst)
        d.list_insert(lst, rnd.randint(0, n), *[rnd.randint(-100, 100) for _ in range(rnd.randint(1, 2))])
    elif r < 0.85:
        n = d.seq_len(lst)
        if n:
            p = rnd.randrange(n)
            d.delete(lst, p, min(rnd.randint(1, 2), n - p))
    elif r < 0.97:
        d.map_set(mp, "k%d" % rnd.randrange(6), rnd.randint(0, 999))
    else:
        d.map_delete(mp, "k%d" % rnd.randrange(6))
    if rnd.random() < 0.3:
        d.commit()


@pytest.mark.parametrize("seed", range(12))
def test_n_site_random_sync_converges(seed):
    """The reference's fuzz strategy (crates/fuzz/src/crdt_fuzzer.rs:223-306): N in-process sites apply
    random actions and sync through update blobs; all sites must converge, a fresh replica that imports
    one full export must agree, and re-export of an imported full history must be byte-identical."""
    rnd = random.Random(seed)
    n_sites = rnd.randint(2, 4)
    docs = [OracleDoc(100 + i) for i in range(n_sites)]
    hs = [(d.get_text("text"), d.get_list("list"), d.get_map("map")) for d in docs]
    for step in range(250):
        i = rnd.randrange(n_sites)
        _random_edit(rnd, docs[i], *hs[i])
        if rnd.random() < 0.08:
            j = rnd.randrange(n_sites)
            if j != i:
                merge(docs[j], docs[i])
    for _ in range(2):
        for i in range(n_sites):
            for j in range(n_sites):
                if i != j:
                    merge(docs[i], docs[j])
    vals = [d.get_deep_value() for d in docs]
    for v in vals[1:]:
        assert v == vals[0]
    assert not any(d.inconsistent_delete() for d in docs)
    full = docs[0].export_updates()
    fresh = OracleDoc(999)
    st = fresh.import_(full)
    assert st["pending"] is None
    assert fresh.get_deep_value() == vals[0]
    assert fresh.oplog_vv() == docs[0].oplog_vv()
    assert fresh.export_updates() == full


from tests.workloads import make_tree_history  # noqa: E402


# ------------------------------------------------------------------ movable tree (SURVEY 8a row a16)
def test_tree_known_answer_loro_rust_test_tree():
    """crates/loro/tests/loro_rust_test.rs:426-444 (`fn tree`): ids, parents, fractional indexes, meta map."""
    d = OracleDoc(1)
    t = d.get_tree("tree")
    root = d.tree_create(t)
    root2 = d.tree_create(t)
    d.tree_move(t, root2, root)
    d.map_set(d.tree_meta(root), "color", "red")
    want = [{"parent": None, "meta": {"color": "red"}, "id": "0@1", "index": 0,
             "children": [{"parent": "0@1", "meta": {}, "id": "1@1", "index": 0, "children": [], "fractional_index": "80"}],
             "fractional_index": "80"}]
    assert d.get_deep_value() == {"tree": want}
    fresh = OracleDoc(7)
    fresh.import_(d.export_updates())
    assert fresh.get_deep_value() == {"tree": want}


def test_tree_known_answer_fractional_indexes():
    """crates/loro/tests/loro_rust_test.rs:1418-1530 (latest version of test_tree_checkout_on_shallow_doc): appended
    siblings get "80" then "8180" (crates/fractional_index/src/lib.rs, jitter 0); ids are the create ops' ids."""
    d = OracleDoc(0)
    t = d.get_tree("tree")
    root = d.tree_create(t)
    c1 = d.tree_create(t)
    d.tree_move(t, c1, root)
    c2 = d.tree_create(t)
    d.tree_move(t, c2, root)
    want = {"tree": [{"parent": None, "meta": {}, "id": "0@0", "index": 0, "fractional_index": "80", "children": [
        {"parent": "0@0", "meta": {}, "id": "1@0", "index": 0, "children": [], "fractional_index": "80"},
        {"parent": "0@0", "meta": {}, "id": "3@0", "index": 1, "children": [], "fractional_index": "8180"}]}]}
    assert d.get_deep_value() == want
    # the intermediate version (checkout to 1@0 in the reference test): two roots "80" / "8180"
    e = OracleDoc(0)
    te = e.get_tree("tree")
    e.tree_create(te)
    e.tree_create(te)
    v = e.get_deep_value()["tree"]
    assert [(n["id"], n["fractional_index"], n["index"]) for n in v] == [("0@0", "80", 0), ("1@0", "8180", 1)]


def test_tree_concurrent_cycle_is_resolved_by_lamport_order():
    """diff_calc/tree.rs:471-508: of two concurrent moves that would form a cycle, the one later in (lamport, peer)
    order is not effected; both replicas agree."""
    a, b = OracleDoc(1), OracleDoc(2)
    ta, tb = a.get_tree("t"), b.get_tree("t")
    x = a.tree_create(ta)
    y = a.tree_create(ta)
    merge(b, a)
    a.tree_move(ta, x, y)       # x under y   (lamport 2, peer 1)
    b.tree_move(tb, y, x)       # y under x   (lamport 2, peer 2) -> would close the cycle: ignored
    merge(a, b)
    merge(b, a)
    va, vb = a.get_deep_value()["t"], b.get_deep_value()["t"]
    assert va == vb
    assert [n["id"] for n in va] == ["1@1"] and [c["id"] for c in va[0]["children"]] == ["0@1"]


def test_tree_delete_hides_subtree_and_move_back_revives():
    a = OracleDoc(1)
    t = a.get_tree("t")
    r = a.tree_create(t)
    k = a.tree_create(t, r)
    g = a.tree_create(t, k)
    a.tree_delete(t, k)
    assert a.get_deep_value()["t"][0]["children"] == []
    b = OracleDoc(2)
    b.import_(a.export_updates())
    assert b.get_deep_value() == a.get_deep_value()
    assert g


@pytest.mark.parametrize("seed", range(8))
def test_tree_random_sites_converge(seed):
    blob, js, vv, docs = make_tree_history(500 + seed, n_sites=2 + seed % 3, n_base=25, n_ops=140, mixed=seed % 2 == 0)
    for d in docs:
        assert d.json_text() == js
    again = OracleDoc(3)
    again.import_(blob)
    assert again.json_text() == js and again.oplog_vv() == vv
    assert again.export_updates() == blob   # re-export of an imported full history is byte-identical


def test_string_arena_growth_model_against_golden_blocks(golden_dir):
    """Whether two adjacent text inserts re-merge depends on the append-only string buffer of the importing document
    (a new buffer generation whenever the cumulative size outgrows the capacity, doubling from 32: arena/str_arena.rs +
    append-only-bytes 0.1.12, not in the tree).  Two peers of the in-tree snapshot `issue_import.base64.txt` typed into
    otherwise idle documents, so their blocks show where the reference's own buffer switched generation: adjacent,
    position-contiguous inserts left UNMERGED at cumulative sizes 32 and 64 (peer 8945398470050628706) and across 64
    (peer 14116964593806747582).  The oracle's model (doc.hpp alloc_str) predicts exactly those cuts."""
    import base64
    import json
    blocks = json.load(open(os.path.join(golden_dir, "snapshot_blocks.json")))
    seqs = {}
    for e in blocks:
        if not e["source"].startswith("issue_import"):
            continue
        d = oracle.decode_dump(base64.b64decode(e["block"]), raw_block=True)
        for b in d.get("blocks", [d] if "changes" in d else []):
            for ch in b["changes"]:
                for op in ch["ops"]:
                    if op["kind"] == "insert_text":
                        seqs.setdefault(ch["peer"], []).append((op["counter"], op["prop"], op["len"], len(op["text"].encode())))
    for peer, cuts in (("8945398470050628706", {32, 64}), ("14116964593806747582", {34})):
        ops = sorted(seqs[peer])
        gens = oracle.i64s(oracle.codec("str_arena_gens", oracle.pack_i64s([o[3] for o in ops])))
        cum, seen = 0, set()
        for (a, ga), (b, gb) in zip(zip(ops, gens), zip(ops[1:], gens[1:])):
            cum += a[3]
            adjacent = b[0] == a[0] + a[2] and b[1] == a[1] + a[2]     # counter- and position-contiguous: mergeable but for the buffer
            if adjacent:
                assert ga != gb, (peer, cum)      # the reference left them apart: the model must put them in different buffers
                seen.add(cum)
        assert seen == cuts, (peer, seen)


def test_map_values_with_nul_bytes_read_back_unchanged():
    """a Str or Binary Map value holding NUL bytes is stored whole (the wrapper passes the payload, not a C string)"""
    d = OracleDoc(5)
    m = d.get_map("m")
    d.map_set(m, "s", "a\x00b\x00")
    d.map_set(m, "b", b"\x00\xff\x00")
    d.map_set(m, "z", b"\x00")
    d.commit()
    want = {"m": {"s": "a\x00b\x00", "b": [0, 255, 0], "z": [0]}}
    assert d.get_deep_value() == want
    e = OracleDoc(6)
    e.import_(d.export_updates())
    assert e.get_deep_value() == want
