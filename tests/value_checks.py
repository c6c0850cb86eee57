"""Value-edge and nesting documents, and the comparisons every one of them goes through: state JSON, vv, frontiers and
status; the re-export (all updates, from versions, in range); JSON updates under both peer-compression settings;
attribution; the state at a mid-history checkout; cursors; a docset that imports the document in two halves.  Shared
by test_values_emu.py and test_values_gpu.py, and by the width cases of width_checks.py.

Each case is one document of two commits by two peers; the first commit is its "middle" (checkout frontiers, the end of
the docset's first half)."""
import random

import loro_b200
from loro_b200 import api
from oracle import CT_LIST, CT_MAP, CT_TEXT, CT_TREE, OracleDoc

from . import json_updates_checks as jc
from . import range_export_checks as rc
from .attribution_checks import attribution_at
from .checkout_checks import json_at, oracle_doc
from .cursor_checks import cursor_pos_ref, sample_cursors, seq_containers
from .engine_checks import check_batch_against_oracle
from .export_checks import check_export_against_oracle, check_export_from_versions

NEST = 64   # LB_MAX_NESTING (include/loro_b200.h)
UNSUPPORTED = 5


class Case:
    def __init__(self, name, blob, mid_frontiers, half1, half2, cursors=()):
        self.name, self.blob, self.mid, self.half1, self.half2 = name, blob, mid_frontiers, half1, half2
        self.cursors = list(cursors)   # [(container, id | None, side)] asked besides the sampled ones


def two_commits(name, first, second, peers=(0x1234, 0xFEDCBA9876543210)):
    """first(doc) and second(doc) edit one document, each in its own commit under its own peer"""
    d = OracleDoc(peers[0])
    first(d)
    d.commit()
    mid, vv1, half1 = d.frontiers(), d.oplog_vv(), d.export_updates()
    d.set_peer_id(peers[1])
    second(d)
    d.commit()
    return Case(name, d.export_updates(), mid, half1, d.export_updates(vv1))


# ---------------------------------------------------------------------------------------------------- scalar edges
I64S = [-2 ** 63, 2 ** 63 - 1, -1, 0, 63, 64, -64, -65, 2 ** 62 - 1, 2 ** 62, -2 ** 62, -2 ** 62 - 1]
F64S = [-0.0, float("nan"), float("inf"), float("-inf"), 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308,
        1e16, 9999999999999998.0, 1e15, 1e-5, 1e-6, 1e-7, 0.1, 123456789012345680.0, -1.5]
SPECIAL = "".join(chr(c) for c in range(0x20)) + "\x7f\"\\ ￿\U0001F99C\U0001D11E"
NAME_SPECIAL = "".join(chr(c) for c in range(1, 0x20)) + "\x7f\"\\ ￿\U0001F99C"   # no NUL in root names


def str_of(n, seed=0):
    """a string of exactly n UTF-8 bytes holding control bytes, quotes, backslashes and multi-byte characters"""
    rnd = random.Random(n * 31 + seed)
    pool = list(SPECIAL) + list("abcxyz 09é語")
    out, size = [], 0
    while size < n:
        ch = rnd.choice(pool)
        b = len(ch.encode())
        if size + b > n:
            ch, b = "a", 1
        out.append(ch)
        size += b
    s = "".join(out)
    assert len(s.encode()) == n
    return s


STR_LENS = [0, 127, 128, 255, 256, 16383, 16384]
BINS = [b"", b"\x00", bytes(range(256)), bytes((7 * i) & 0xFF for i in range(300))]


def scalar_cases():
    def ints_a(d):
        d.list_insert(d.get_list("l"), 0, *I64S)
        m = d.get_map("m")
        for k, v in enumerate(I64S):
            d.map_set(m, "i%d" % k, v)

    def ints_b(d):
        d.list_insert(d.get_list("l"), 3, *reversed(I64S))
        d.map_set(d.get_map("m"), "i0", 2 ** 63 - 1)

    def floats_a(d):
        d.list_insert(d.get_list("l"), 0, *F64S)
        m = d.get_map("m")
        for k, v in enumerate(F64S):
            d.map_set(m, "f%d" % k, v)

    def floats_b(d):
        d.list_insert(d.get_list("l"), 1, -0.0, float("nan"))
        d.map_set(d.get_map("m"), "f1", 5e-324)

    def strs_a(d):
        l, m, t = d.get_list("l"), d.get_map("m"), d.get_text("t")
        for n in STR_LENS:
            d.list_insert(l, d.seq_len(l), str_of(n))
            d.map_set(m, "s%d" % n, str_of(n, 1))
        d.map_set(m, "", str_of(5, 2))                       # the empty key
        d.map_set(m, SPECIAL, 1)                             # a key of every escaped character
        d.map_set(m, str_of(300, 3), "long key")
        d.text_insert(t, 0, SPECIAL + str_of(200, 4))

    def strs_b(d):
        l, m, t = d.get_list("l"), d.get_map("m"), d.get_text("t")
        d.list_insert(l, 2, SPECIAL, "", "\U0001F99C")
        d.map_set(m, "", "")
        d.map_set(m, "s128", str_of(16384, 5))
        d.text_insert(t, 3, "\U0001F99C\x00 ")
        d.map_set(d.get_map(NAME_SPECIAL), "k", SPECIAL)     # a root container named with escaped characters
        d.list_insert(d.get_list("\U0001D11E"), 0, 1)

    def bins_a(d):
        d.list_insert(d.get_list("l"), 0, *BINS)
        m = d.get_map("m")
        for k, v in enumerate(BINS):
            d.map_set(m, "b%d" % k, v)

    def bins_b(d):
        d.list_insert(d.get_list("l"), 2, b"\x00", b"")
        d.map_set(d.get_map("m"), "b2", b"\x00" * 3)

    def lists_a(d):
        l = d.get_list("l")
        d.list_insert(l, 0, "one")
        d.list_insert(l, 0, *range(8))                       # the warp decoder's item limit
        d.list_insert(l, 8, *range(100, 109))                # one past it
        d.list_insert(l, 0, *["s%d" % i for i in range(9)])

    def lists_b(d):
        l = d.get_list("l")
        d.list_insert(l, 4, *[1.5] * 8)
        d.list_insert(l, 0, *[b"\x01"] * 9)

    def child_keys_a(d):
        m = d.get_map("m")
        c = d.map_set_container(m, SPECIAL, CT_MAP)          # child-container keys
        d.map_set(c, "\U0001F99C", "\x00")
        c2 = d.map_set_container(m, "", CT_TEXT)
        d.text_insert(c2, 0, SPECIAL)

    def child_keys_b(d):
        m = d.get_map("m")
        c = d.map_set_container(m, str_of(200, 6), CT_LIST)
        d.list_insert(c, 0, str_of(256, 7), b"\x00")

    return [two_commits("i64", ints_a, ints_b), two_commits("f64", floats_a, floats_b),
            two_commits("str", strs_a, strs_b), two_commits("binary", bins_a, bins_b),
            two_commits("list-items", lists_a, lists_b), two_commits("child-keys", child_keys_a, child_keys_b)]


def composite_cases():
    def wide_map_a(d):
        big = {"key%03d" % i: i for i in range(140)}         # > 127 keys: two-byte key indices inside the value
        d.list_insert(d.get_list("l"), 0, big, [big, {"x": big}])
        d.map_set(d.get_map("m"), "big", big)

    def wide_map_b(d):
        d.map_set(d.get_map("m"), "other", {"key139": "last", "\U0001F99C": {"": None}, SPECIAL: [b"\x00", -0.0]})

    def containers_a(d):
        l, m = d.get_list("l"), d.get_map("m")
        for ct in (CT_MAP, CT_LIST, CT_TEXT, CT_TREE):
            d.list_insert_container(l, 0, ct)
        t = d.map_set_container(m, "text", CT_TEXT)
        d.text_insert(t, 0, "inner")
        sub = d.list_insert_container(l, 2, CT_MAP)
        d.map_set(sub, "k", [1, {"a": b"\x00"}])
        tr = d.map_set_container(m, "tree", CT_TREE)
        n = d.tree_create(tr)
        d.map_set(d.tree_meta(n), "title", SPECIAL)

    def containers_b(d):
        m = d.get_map("m")
        lst = d.map_set_container(m, "list", CT_LIST)
        d.list_insert(lst, 0, {"deep": [[[1]]]}, "x")
        d.map_set(m, "text", "overwritten")

    return [two_commits("wide-map", wide_map_a, wide_map_b), two_commits("containers", containers_a, containers_b)]


def warp_edge_cases():
    """values whose encoded length is 255 / 256 bytes (the warp decoder's lane-parallel limit), values straddling its
    144-byte chunk edges, and values sections just under and just over DW_VALS = 4608 bytes.  Every commit is one
    change of one peer, so one block whose values are all of one kind."""
    def map_sets(name, sizes):
        """Map sets whose encoded values (kind byte, two-byte length, bytes) are `sizes` bytes long"""
        def f(d):
            m = d.get_map(name)
            for k, n in enumerate(sizes):
                d.map_set(m, "v%03d" % k, ("%d" % (k % 10)) * (n - 3))
        return f

    def section(total):
        sizes, left = [], total
        while left:
            take = 203 if left - 203 >= 131 or left == 203 else left
            sizes.append(take)
            left -= take
        return sizes

    def text_255(d):
        d.text_insert(d.get_text("t"), 0, "z" * 253)   # varint(253) + 253 bytes

    return [two_commits("len-255-then-256", map_sets("m", [255, 131, 255]), map_sets("n", [256, 140])),
            two_commits("chunk-edges", map_sets("m", [103] * 40 + [145] * 9), text_255),
            two_commits("section-under-over", map_sets("w", section(4600)), map_sets("x", section(4620)))]


# ---------------------------------------------------------------------------------------------------- nesting
def nested_value(levels, leaf=1):
    """a LoroValue `levels` List / Map levels deep (the outermost counts), alternating [ and {"k": ...}"""
    v = leaf
    for i in range(levels):
        v = [v] if i % 2 == 0 else {"k": v}
    return v


def container_chain(d, root_kind, kinds, levels):
    """`levels` child containers below a root container of `root_kind`, each the only child of the one above, the kinds
    taken in turn from `kinds`; returns (innermost container, its kind)"""
    c = d.get_map("root") if root_kind == CT_MAP else d.get_list("root")
    kind = root_kind
    for i in range(levels):
        ck = kinds[i % len(kinds)]
        c = d.map_set_container(c, "c", ck) if kind == CT_MAP else d.list_insert_container(c, 0, ck)
        kind = ck
    return c, kind


def put_deep(d, c, kind, levels):
    """a value `levels` levels deep into container c: a Map set, or a List insert (whose own List is one level)"""
    if kind == CT_MAP:
        d.map_set(c, "v", nested_value(levels))
    else:
        d.list_insert(c, d.seq_len(c), nested_value(levels - 1))


def chain_case(name, root_kind, kinds, levels, value_levels=0):
    """a chain of `levels` child containers; the innermost holds one int, or a value `value_levels` deep"""
    def first(d):
        c, k = container_chain(d, root_kind, kinds, levels)
        if value_levels:
            put_deep(d, c, k, value_levels)
        elif k == CT_MAP:
            d.map_set(c, "v", 7)
        else:
            d.list_insert(c, 0, 7)

    def second(d):
        d.map_set(d.get_map("side"), "k", 1)
    return two_commits(name, first, second)


def value_case(name, kind, levels):
    """one List insert (the insert's own List is one level) or Map set of a value `levels` levels deep"""
    def first(d):
        put_deep(d, d.get_list("l") if kind == CT_LIST else d.get_map("m"), kind, levels)

    def second(d):
        if kind == CT_LIST:
            d.list_insert(d.get_list("l"), 1, nested_value(levels - 1, leaf="x"))
        else:
            d.map_set(d.get_map("m"), "w", nested_value(levels, leaf="x"))
    return two_commits(name, first, second)


def depth_cases(levels):
    """documents nested exactly `levels` deep (NEST: at the bound, NEST + 1: one past it): container chains of every
    shape, deep values in List inserts and Map sets, and both at once"""
    return [chain_case("map-chain", CT_MAP, [CT_MAP], levels),
            chain_case("list-chain", CT_LIST, [CT_LIST], levels),
            chain_case("alternating-chain", CT_MAP, [CT_LIST, CT_MAP], levels),
            value_case("list-value", CT_LIST, levels),
            value_case("map-value", CT_MAP, levels),
            chain_case("deep-list-chain-deep-value", CT_LIST, [CT_LIST], levels, value_levels=NEST),
            chain_case("deep-map-chain-deep-value", CT_MAP, [CT_MAP, CT_LIST], NEST, value_levels=levels)]


# ---------------------------------------------------------------------------------------------------- comparisons
def check_cases(cases, lib_path=None):
    """every output of every case against the reference, byte for byte"""
    blobs = [c.blob for c in cases]
    check_batch_against_oracle(blobs, lib_path=lib_path)
    check_export_against_oracle(blobs, lib_path=lib_path)
    refs = [oracle_doc([b]) for b in blobs]
    for k, b in enumerate(blobs):
        check_export_from_versions(b, lib_path=lib_path, seed=k, trials=3)
    batch = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT | api.LB_FLAG_ATTRIBUTION, lib_path=lib_path)
    rnd = random.Random(5)
    reqs = []
    for k, r in enumerate(refs):
        vv = r.oplog_vv()
        reqs += [(k, rc.till_spans(vv)), (k, [(p, rnd.randint(0, c), c) for p, c in vv.items()])]
    rc.check_requests(batch, refs, reqs, single=False)
    ranges = []
    for k, r in enumerate(refs):
        ranges += [(k, None, None), (k,) + jc.random_range(rnd, r.oplog_vv())]
    jc.compare_batch(batch, refs, ranges)
    for k, r in enumerate(refs):
        assert batch.attribution_bytes(k) == attribution_at(r), cases[k].name
    at = loro_b200.import_batch_at(blobs, {k: c.mid for k, c in enumerate(cases)}, lib_path=lib_path)
    for k, (c, r) in enumerate(zip(cases, refs)):
        assert at.status(k).code == 0, (c.name, at.status(k))
        assert at.json_bytes(k) == json_at(r, c.mid), c.name
    answers = check_cursors(cases, refs, lib_path)
    check_docset_halves(cases, lib_path)
    return answers


def check_cursors(cases, refs, lib_path=None, k=80):
    """k cursors sampled over every Text / List container of each case, and the case's own cursors, against the
    reference field by field; returns each case's [(cursor, answer)]"""
    batch = loro_b200.import_batch([c.blob for c in cases], flags=api.LB_FLAG_CURSORS, lib_path=lib_path)
    rnd = random.Random(9)
    reqs, want = [], []
    for i, (c, r) in enumerate(zip(cases, refs)):
        cids = sorted(seq_containers(r))
        cs = (sample_cursors(rnd, cids, r.oplog_vv(), k) if cids else []) + c.cursors
        reqs += [(i,) + x for x in cs]
        want += cursor_pos_ref(r, cs)
    got = batch.cursor_pos(reqs)
    bad = [(cases[q[0]].name, q, g, w) for q, g, w in zip(reqs, got, want) if g != w]
    assert not bad, (len(bad), bad[:6])
    out = [[] for _ in cases]
    for q, g in zip(reqs, got):
        out[q[0]].append((q[1:], g))
    return out


def check_docset_halves(cases, lib_path=None):
    """a docset document per case takes the first half, then the second: after each, the reference's state, vv and
    export"""
    ds = loro_b200.DocSet(lib_path=lib_path)
    refs = [OracleDoc(0xD0C) for _ in cases]
    for half in (0, 1):
        r = ds.import_([c.half2 if half else c.half1 for c in cases], list(range(len(cases))), flags=api.LB_FLAG_EXPORT)
        for k, (c, ref) in enumerate(zip(cases, refs)):
            ref.import_(c.half2 if half else c.half1)
            assert r.status(k).code == 0, (c.name, half, r.status(k))
            assert r.json_bytes(k) == ref.json_text(), (c.name, half)
            assert r.oplog_vv(k) == ref.oplog_vv(), (c.name, half)
            assert r.export_updates(k) == ref.export_updates(), (c.name, half)
        r.close()
    ds.close()


def check_past_bound(cases, lib_path=None):
    """documents nested one level past LB_MAX_NESTING: UNSUPPORTED on plain import, at a checkout and in a docset (the
    reference imports them; the engine does not cover them), never DECODE or CAPACITY"""
    blobs = [c.blob for c in cases]
    b = loro_b200.import_batch(blobs, lib_path=lib_path)
    e = loro_b200.import_batch(blobs, flags=api.LB_FLAG_EXPORT, lib_path=lib_path)
    at = loro_b200.import_batch_at(blobs, {k: c.mid for k, c in enumerate(cases)}, lib_path=lib_path)
    for k, c in enumerate(cases):
        OracleDoc(1).import_(c.blob)                       # well-formed: the reference's import succeeds
        assert b.status(k).code == UNSUPPORTED, (c.name, b.status(k))
        assert e.status(k).code == UNSUPPORTED, (c.name, e.status(k))
        assert at.status(k).code == UNSUPPORTED, (c.name, at.status(k))
        assert b.json_bytes(k) == b"", c.name
    ds = loro_b200.DocSet(lib_path=lib_path)
    r = ds.import_([c.blob for c in cases], list(range(len(cases))))
    for k, c in enumerate(cases):
        assert r.status(k).code == UNSUPPORTED, (c.name, r.status(k))
    r.close()
    ds.close()
