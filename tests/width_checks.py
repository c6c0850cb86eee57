"""Documents past the per-document widths of the warp-per-document kernels: the peer tables of the attribution writer
(ATTR_SMEM_PEERS) and of the parallel tree writer (TREE_TXT_PEERS), the 32-lane ballot rounds over peers and containers,
the container and key sorts, the 32-way span search of cursors, and fractional indexes longer than the tree writer's
lane buffer takes.  Each builder measures, on the reference, the width its document reaches and asserts it, so that a
change to a generator cannot drop a case below its threshold; every case goes through value_checks.check_cases.
Shared by test_widths_emu.py and test_widths_gpu.py."""
import json
import random

from oracle import CT_LIST, CT_MAP, CT_TEXT, OracleDoc

from . import workloads
from .attribution_checks import attribution_at
from .cursor_checks import seq_containers
from .test_large_batch_gpu import csrc_define
from .value_checks import Case

TREE_TXT_PEERS = csrc_define("k_state.cuh", "TREE_TXT_PEERS")    # the parallel tree writer's shared peer table
ATTR_SMEM_PEERS = csrc_define("k_attr.cuh", "ATTR_SMEM_PEERS")   # the attribution writer's shared peer table
WARP = 32                                                         # one ballot round, one level of the span search


def reference(blob):
    d = OracleDoc(1)
    d.import_(blob)
    return d


def attribution(doc):
    return json.loads(attribution_at(doc))["containers"]


def width_case(name, blob, mid, half1, half2, width, cursors=(), cover=None):
    """a value_checks.Case that also carries the width it reached on the reference, e.g. "P=33" or "spans=1025", and
    cover: (peers, Text / List containers) that its own cursors find targets of"""
    c = Case(name, blob, mid, half1, half2, cursors)
    c.width, c.cover = width, cover
    return c


def peer_ids(rnd, n, low=1):
    """n distinct peer ids: `low` (0 or 1) and random ids alternately from the lower and the upper half of the u64 range"""
    ids = [low]
    while len(ids) < n:
        p = rnd.getrandbits(63) | ((len(ids) & 1) << 63)
        if p not in ids:
            ids.append(p)
    rnd.shuffle(ids)
    return ids


def sync_all(docs):
    """every replica ends with every change: all into docs[0], then docs[0] into the others"""
    for d in docs:
        d.commit()
    for d in docs[1:]:
        workloads.merge(docs[0], d)
    for d in docs[1:]:
        workloads.merge(d, docs[0])


def concurrent_history(name, peers, first, second):
    """first(k, doc) and second(k, doc) run on every peer's replica without syncing in between (concurrent edits);
    everything is synced after each round.  The end of the first round is the case's middle."""
    docs = [OracleDoc(p) for p in peers]
    for k, d in enumerate(docs):
        first(k, d)
    sync_all(docs)
    col = docs[0]
    mid, vv1, half1 = col.frontiers(), col.oplog_vv(), col.export_updates()
    for k, d in enumerate(docs):
        second(k, d)
    sync_all(docs)
    return col.export_updates(), mid, half1, col.export_updates(vv1)


def every_id_cursors(doc, cids, cap=3000):
    """a cursor at every id of the oplog in every given container, the side cycling: visible and deleted elements of
    each peer, and ids that are not elements of that container (a fixed sample of `cap` of them when there are more)"""
    out = []
    for cid in sorted(cids):
        for p, n in sorted(doc.oplog_vv().items()):
            for c in range(n):
                out.append((cid, (p, c), (c % 3) - 1))
    return out if len(out) <= cap else random.Random(len(out)).sample(out, cap)


def near_id_cursors(doc, radius=3):
    """cursors at the visible elements of every Text / List container and at the ids up to `radius` counters either
    side of them (the deleted elements of the same inserts among them), the side cycling"""
    out = set()
    for cid, ids in seq_containers(doc).items():
        for p, c in ids:
            out.update((cid, (p, x), (x % 3) - 1) for x in range(max(0, c - radius), c + radius + 1))
    return sorted(out)


def check_coverage(cases, answers):
    """the cases' own cursors reach what they are there for: deleted targets, and found targets of every peer and every
    Text / List container the case names in `cover`"""
    for c, ans in zip(cases, answers):
        if not c.cursors:
            continue
        found = [(q, g) for q, g in ans if g[0] == 0 and q[1] is not None]
        peers, cids = {q[1][0] for q, _ in found}, {q[0] for q, _ in found}
        deleted = sum(1 for _, g in found if g[3] is not None)
        print(c.name, "cursors: %d found, %d deleted targets, %d peers, %d containers" %
              (len(found), deleted, len(peers), len(cids)))
        assert deleted and (len(peers), len(cids)) == c.cover, (c.name, deleted, len(peers), len(cids), c.cover)


def seq_cids(doc):
    return [cid for cid in attribution(doc) if cid.endswith(":Text") or cid.endswith(":List")]


# ---------------------------------------------------------------------------------------------------- peers
def peer_case(n_peers, low=1):
    """n_peers concurrent sites, every one inserting into Text, List and Map and deleting from them"""
    rnd = random.Random(1000 + n_peers)
    peers = peer_ids(rnd, n_peers, low)

    def first(k, d):
        t, l, m = d.get_text("text"), d.get_list("list"), d.get_map("map")
        d.text_insert(t, rnd.randint(0, d.seq_len(t)), "p%d." % k)
        d.list_insert(l, rnd.randint(0, d.seq_len(l)), k, "s%d" % k)
        d.map_set(m, "k%d" % (k % 40), k)
        for _ in range(3):
            workloads.random_edit(rnd, d, t, l, m)

    def second(k, d):
        t, l, m = d.get_text("text"), d.get_list("list"), d.get_map("map")
        for c in (t, l):
            n = d.seq_len(c)
            if n > 1:
                d.delete(c, rnd.randrange(n - 1), 2)
        d.map_delete(m, "k%d" % ((k * 7) % 40))
        d.text_insert(t, rnd.randint(0, d.seq_len(t)), "q%d" % k)
        workloads.random_edit(rnd, d, t, l, m)

    blob, mid, h1, h2 = concurrent_history("peers", peers, first, second)
    ref = reference(blob)
    vv = ref.oplog_vv()
    assert len(vv) == n_peers and low in vv and any(p >> 63 for p in vv) and any(p and not p >> 63 for p in vv), vv
    cids = seq_cids(ref)
    return width_case("peers-%d" % n_peers, blob, mid, h1, h2, "P=%d" % len(vv), every_id_cursors(ref, cids),
                      (n_peers, len(cids)))


def peer_cases():
    widths = sorted({TREE_TXT_PEERS, TREE_TXT_PEERS + 1, ATTR_SMEM_PEERS, ATTR_SMEM_PEERS + 1, 2 * WARP, 2 * WARP + 1})
    return [peer_case(n, low=0 if n == TREE_TXT_PEERS + 1 else 1) for n in widths]


# ---------------------------------------------------------------------------------------------------- trees
def tree_json_nodes(doc_json, root="tree"):
    """every node of a tree in the reference's state JSON, depth first"""
    out, stack = [], list(json.loads(doc_json)[root])
    while stack:
        n = stack.pop()
        out.append(n)
        stack += n["children"]
    return out


def tree_case(n_peers, meta=False, fi_zigzag=0):
    """n_peers sites create nodes under each other's nodes, then move and delete them concurrently; with `meta`, some
    nodes get meta map entries (the serial tree writer), otherwise none does (the parallel one).  fi_zigzag > 0: one
    site creates that many children of one parent alternately just before and just after the last one it created,
    which lengthens their fractional index by a byte a create."""
    rnd = random.Random(2000 + n_peers + 100 * meta + fi_zigzag)
    peers = peer_ids(rnd, n_peers)
    p_meta = 0.2 if meta else 0.0
    docs = [OracleDoc(p) for p in peers]
    base, tr0 = docs[0], docs[0].get_tree("tree")
    for _ in range(12):                   # a base tree that every site has before they edit concurrently
        workloads.random_tree_edit(rnd, base, tr0, p_create=1.0, p_meta=p_meta)
    if fi_zigzag:                         # a second tree: the long fractional indexes, out of the churn's reach
        fi_tree = base.get_tree("fi")
        parent, last = base.tree_create(fi_tree), 0
        base.tree_create(fi_tree, parent)
        for j in range(fi_zigzag):
            last += j % 2
            base.tree_create(fi_tree, parent, last)
    base.commit()
    for d in docs[1:]:
        workloads.merge(d, base)

    def grow(k, d):
        tr = d.get_tree("tree")
        for _ in range(2):
            nodes = d.tree_nodes(tr)
            d.tree_create(tr, rnd.choice(nodes), -1 if rnd.random() < 0.5 else 0)
        if fi_zigzag:                     # siblings of the long indexes from every site, concurrently
            d.tree_create(d.get_tree("fi"), parent, 1 + k % 5)
        if meta and k % 3 == 0:
            d.map_set(d.tree_meta(rnd.choice(d.tree_nodes(tr))), "k%d" % (k % 4), k)

    def churn(k, d):
        tr = d.get_tree("tree")
        for _ in range(3):
            workloads.random_tree_edit(rnd, d, tr, p_create=0.25, p_delete=0.06, p_meta=p_meta)

    for _ in range(2):                    # the second round creates children of the other sites' nodes
        for k, d in enumerate(docs):
            grow(k, d)
        sync_all(docs)
    col = docs[0]
    mid, vv1, h1 = col.frontiers(), col.oplog_vv(), col.export_updates()
    for k, d in enumerate(docs):
        churn(k, d)
    sync_all(docs)
    blob = col.export_updates()
    ref = reference(blob)
    vv = ref.oplog_vv()
    nodes = tree_json_nodes(ref.json_text())
    fi_nodes = tree_json_nodes(ref.json_text(), "fi") if fi_zigzag else []
    nodes += fi_nodes
    with_meta = sum(1 for n in nodes if n["meta"])
    assert len(vv) == n_peers, vv
    assert (with_meta > 0) == meta, with_meta
    # node ids and parents of nodes created by many peers, so the writer formats them from every slot of its peer table
    id_peers = len({n["id"].split("@")[1] for n in nodes})
    parent_peers = len({n["parent"].split("@")[1] for n in nodes if n["parent"]})
    assert id_peers >= min(n_peers, TREE_TXT_PEERS + 1) and parent_peers >= min(n_peers, TREE_TXT_PEERS + 1) // 2, \
        (id_peers, parent_peers)
    width = "P=%d %s" % (len(vv), "meta" if meta else "no-meta")
    if fi_zigzag:
        fi = sorted(len(n["fractional_index"]) // 2 for n in fi_nodes)
        assert len({n["id"].split("@")[1] for n in fi_nodes}) == n_peers
        assert 32 in fi and max(fi) > 32, fi
        width += " fi-bytes=%d" % max(fi)
    name = "tree-%d%s%s" % (n_peers, "-meta" if meta else "", "-fi" if fi_zigzag else "")
    return width_case(name, blob, mid, h1, col.export_updates(vv1), width)


def tree_cases():
    T = TREE_TXT_PEERS
    return ([tree_case(n) for n in (T, T + 1, WARP + 1, 40)] + [tree_case(T + 4, meta=True)] +
            [tree_case(3, fi_zigzag=60), tree_case(T + 2, fi_zigzag=60)])


# ---------------------------------------------------------------------------------------------------- containers
def container_case(n):
    """n containers in one document, half roots and half children of a root Map and a root List, the kinds Text / List /
    Map in turn; root names sort in the reverse of their creation order.  A second peer then deletes from and inserts
    into every Text and List, and sets a key of every Map."""
    kinds = (CT_TEXT, CT_LIST, CT_MAP)
    made = []   # (handle, kind) in creation order

    def fill(d, c, kind, tag):
        if kind == CT_TEXT:
            d.text_insert(c, 0, "%s-text" % tag)
        elif kind == CT_LIST:
            d.list_insert(c, 0, tag, 1, 2.5)
        else:
            d.map_set(c, "k", tag)

    def first(d):
        hub, hubl = d.get_map("hub"), d.get_list("hubl")
        n_roots = n // 2 - 2
        for k in range(n_roots):
            kind = kinds[k % 3]
            c = d.container("r%03d" % (n_roots - k), kind)
            fill(d, c, kind, "r%d" % k)
            made.append((c, kind))
        for k in range(n - n_roots - 2):
            kind = kinds[k % 3]
            c = d.map_set_container(hub, "c%03d" % k, kind) if k % 2 else d.list_insert_container(hubl, 0, kind)
            fill(d, c, kind, "c%d" % k)
            made.append((c, kind))

    def second(d):
        for k, (c, kind) in enumerate(made):
            if kind == CT_MAP:
                d.map_set(c, "j", k)
            else:
                d.delete(c, 1, 2)
                (d.text_insert(c, 1, "+") if kind == CT_TEXT else d.list_insert(c, 1, k))

    d = OracleDoc(0x51)
    first(d)
    d.commit()
    mid, vv1, h1 = d.frontiers(), d.oplog_vv(), d.export_updates()
    d.set_peer_id(0xF00D00000000051)
    second(d)
    d.commit()
    blob = d.export_updates()
    ref = reference(blob)
    conts = attribution(ref)
    assert len(conts) == n, (n, sorted(conts))
    return width_case("containers-%d" % n, blob, mid, h1, d.export_updates(vv1), "C=%d" % len(conts),
                      near_id_cursors(ref), (2, len(seq_cids(ref))))


def container_cases():
    return [container_case(n) for n in (WARP - 1, WARP, WARP + 1, 2 * WARP, 2 * WARP + 1)]


# ---------------------------------------------------------------------------------------------------- keys
def key_names(n, seed):
    """n distinct keys of different lengths whose byte order is not their order here"""
    rnd = random.Random(seed)
    names = ["", "~"] + ["%s%d" % ("k" * (1 + i % 3), (i * 37) % 97) for i in range(n)]
    names = list(dict.fromkeys(names))[:n]
    rnd.shuffle(names)
    return names


def key_case(name, maps):
    """maps: {root map name: its keys}.  The first site sets every key; then it and a second site concurrently
    overwrite and delete the keys past the first 32 in byte order."""
    d = OracleDoc(0xAB)
    for mname, keys in maps.items():
        m = d.get_map(mname)
        for i, k in enumerate(keys):
            d.map_set(m, k, i)
    d.commit()
    mid, vv1, h1 = d.frontiers(), d.oplog_vv(), d.export_updates()
    e = OracleDoc(0x8000000000000AB0)
    e.import_(h1)
    for mname, keys in maps.items():
        late = sorted(keys, key=lambda k: k.encode())[WARP - 2:]
        for i, k in enumerate(late):
            if i % 2:
                e.map_delete(e.get_map(mname), k)
            else:
                e.map_set(e.get_map(mname), k, "e%d" % i)
            if i % 3 == 0:
                d.map_set(d.get_map(mname), k, "d%d" % i)
            elif i % 3 == 1:
                d.map_delete(d.get_map(mname), k)
    d.commit()
    e.commit()
    workloads.merge(d, e)
    blob = d.export_updates()
    ref = reference(blob)
    conts = attribution(ref)
    per_map = {m: len(conts["cid:root-%s:Map" % m]) for m in maps}
    assert per_map == {m: len(set(ks)) for m, ks in maps.items()}, per_map
    distinct = len(set(k for ks in maps.values() for k in ks))
    return width_case(name, blob, mid, h1, d.export_updates(vv1), "K=%d %s" % (distinct, per_map))


def key_cases():
    out = [key_case("keys-%d" % n, {"m": key_names(n, n)}) for n in (WARP - 1, WARP, WARP + 1, 2 * WARP + 1)]
    spread = {"a": key_names(20, 1), "b": key_names(30, 2), "c": key_names(45, 3)[15:], "d": ["only-%d" % i for i in range(9)]}
    return out + [key_case("keys-spread", spread)]


# ---------------------------------------------------------------------------------------------------- spans
SPAN_EDGES = (0, 1, 2, WARP - 2, WARP - 1, WARP, WARP + 1, WARP * WARP - 2, WARP * WARP - 1, WARP * WARP,
              WARP * WARP + 1, WARP ** 3 - 2, WARP ** 3 - 1, WARP ** 3, WARP ** 3 + 1)


def span_case(name, sizes):
    """sizes: {(root name, kind): n}.  One site types each container right to left, an element an op, so its rope holds
    exactly n spans, one per element (no element continues the one before it); a second site then deletes every third
    element and the elements on both sides of each 32-way search boundary, counted from either end."""
    a = OracleDoc(0x5A)
    conts = {}
    for (cname, kind), n in sizes.items():
        c = a.container(cname, kind)
        base = a.oplog_vv().get(0x5A, 0)
        for i in range(n):
            if kind == CT_TEXT:
                a.text_insert(c, 0, "abcdefghij"[i % 10])
            else:
                a.list_insert(c, 0, i)
        conts[(cname, kind)] = (c, base)
    a.commit()
    mid, vv1, h1 = a.frontiers(), a.oplog_vv(), a.export_updates()
    b = OracleDoc(0xE5)
    b.import_(h1)
    cursors = []
    for (cname, kind), n in sizes.items():
        c, base = conts[(cname, kind)]
        cid = "cid:root-%s:%s" % (cname, "Text" if kind == CT_TEXT else "List")
        edges = {e for e in SPAN_EDGES if e < n} | {n - 1 - e for e in SPAN_EDGES if e < n}
        # document position j holds the element of counter base + n - 1 - j; deleting from the end keeps the positions
        # before the deleted one
        gone = sorted({j for j in range(0, n, 3)} | {j for j in edges if j % 4 != 1}, reverse=True)
        for j in gone:
            b.delete(b.container(cname, kind), j, 1)
        for e in sorted(edges):
            cursors += [(cid, (0x5A, base + e), side) for side in (-1, 0, 1)]
    b.commit()
    workloads.merge(a, b)
    blob = a.export_updates()
    ref = reference(blob)
    got = attribution(ref)
    widths = []
    for (cname, kind), n in sizes.items():
        c, base = conts[(cname, kind)]
        cid = "cid:root-%s:%s" % (cname, "Text" if kind == CT_TEXT else "List")
        runs = got[cid]
        # every visible element is a run of its own, counters falling: no two elements of the rope make one span
        assert all(r[2] == 1 for r in runs) and all(x[1] > y[1] for x, y in zip(runs, runs[1:])), cid
        assert ref.oplog_vv()[0x5A] >= base + n and 0 < len(runs) < n, (cid, len(runs))
        widths.append("spans=%d" % n)
    return width_case(name, blob, mid, h1, a.export_updates(vv1), " ".join(widths), cursors, (1, len(sizes)))


def span_cases():
    small = {("t%d" % n, CT_TEXT): n for n in (WARP - 1, WARP, WARP + 1)}
    small.update({("l%d" % n, CT_LIST): n for n in (WARP - 1, WARP, WARP + 1)})
    mid = {("t1024", CT_TEXT): WARP * WARP, ("l1025", CT_LIST): WARP * WARP + 1}
    return [span_case("spans-small", small), span_case("spans-1024", mid),
            span_case("spans-32769", {("t32769", CT_TEXT): WARP ** 3 + 1})]


def all_cases():
    return peer_cases() + tree_cases() + container_cases() + key_cases() + span_cases()
