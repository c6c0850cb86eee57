"""Seeded multi-site workloads built with the oracle (test infrastructure).

Mirrors the reference's fuzz strategy (crates/fuzz/src/crdt_fuzzer.rs): N in-process sites apply random
actions to Text/List/Map containers and sync through FastUpdates blobs.  Returns the full-history blob that
`export(all_updates)` of a fully synced replica yields plus the oracle's expected results.
"""
import random

import oracle
from oracle import OracleDoc


def merge(a, b):
    return a.import_(b.export_updates(a.oplog_vv()))


def random_child_edit(rnd, d, lst, mp):
    """Child containers (handler.rs insert_container): created inside the root map or list, then edited like roots;
    state.rs:1039 get_container_deep_value inlines them in the parent's JSON."""
    if not hasattr(d, "_kids"):
        d._kids = []   # child container handles this site created
    kids = d._kids
    if not kids or rnd.random() < 0.3:
        ctype = rnd.choice([oracle.CT_TEXT, oracle.CT_LIST, oracle.CT_MAP])
        if rnd.random() < 0.5:
            h = d.map_set_container(mp, "c%d" % rnd.randrange(6), ctype)
        else:
            h = d.list_insert_container(lst, rnd.randint(0, d.seq_len(lst)), ctype)
        kids.append((h, ctype))
        return
    h, ctype = rnd.choice(kids)
    if ctype == oracle.CT_TEXT:
        d.text_insert(h, rnd.randint(0, d.seq_len(h)), "".join(rnd.choice("child xyz") for _ in range(rnd.randint(1, 4))))
    elif ctype == oracle.CT_LIST:
        if rnd.random() < 0.2 and len(kids) < 12:   # a grandchild
            kids.append((d.list_insert_container(h, rnd.randint(0, d.seq_len(h)), oracle.CT_MAP), oracle.CT_MAP))
        else:
            d.list_insert(h, rnd.randint(0, d.seq_len(h)), rnd.randint(0, 9))
    else:
        d.map_set(h, "k%d" % rnd.randrange(3), rnd.randint(0, 99))


def random_edit(rnd, d, text, lst, mp, weights=(0.35, 0.15, 0.25, 0.10, 0.12, 0.03), unicode_=True, children=0.04):
    if children and rnd.random() < children:
        return random_child_edit(rnd, d, lst, mp)
    r = rnd.random()
    w = weights
    alphabet = "abcdefg xyz\"\\\n" + ("é中😀" if unicode_ else "")
    if r < w[0]:
        n = d.seq_len(text)
        d.text_insert(text, rnd.randint(0, n), "".join(rnd.choice(alphabet) for _ in range(rnd.randint(1, 5))))
    elif r < w[0] + w[1]:
        n = d.seq_len(text)
        if n:
            p = rnd.randrange(n)
            d.delete(text, p, min(rnd.randint(1, 4), n - p))
    elif r < w[0] + w[1] + w[2]:
        n = d.seq_len(lst)
        vals = []
        for _ in range(rnd.randint(1, 3)):
            k = rnd.random()
            if k < 0.6:
                vals.append(rnd.randint(-2**40, 2**40) if rnd.random() < 0.2 else rnd.randint(-100, 100))
            elif k < 0.85:
                vals.append("".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 8))))
            elif k < 0.9:
                vals.append(None)
            elif k < 0.95:
                vals.append(rnd.random() < 0.5)
            elif k < 0.98:
                vals.append(rnd.choice([float(rnd.randint(-1000, 1000)), rnd.uniform(-1e3, 1e3), rnd.random() * 10.0 ** rnd.randint(-12, 25)]))
            else:   # nested LoroValue::List / Map (keys index the block's key arena on the wire)
                vals.append(rnd.choice([{"n%d" % rnd.randrange(3): rnd.randint(0, 9), "m": {"deep": [1, {"x": None}]}}, [1, [2.5, "s"], {}]]))
        d.list_insert(lst, rnd.randint(0, n), *vals)
    elif r < w[0] + w[1] + w[2] + w[3]:
        n = d.seq_len(lst)
        if n:
            p = rnd.randrange(n)
            d.delete(lst, p, min(rnd.randint(1, 4), n - p))
    elif r < 1 - w[5]:
        r2 = rnd.random()
        v = rnd.randint(0, 999) if r2 < 0.75 else ("v%d" % rnd.randrange(9) if r2 < 0.9 else
                                                   (rnd.uniform(-5, 5) if r2 < 0.95 else {"a": [rnd.randint(0, 3)], "k%d" % rnd.randrange(16): {"b": 0.5}}))
        d.map_set(mp, "k%d" % rnd.randrange(16), v)
    else:
        d.map_delete(mp, "k%d" % rnd.randrange(16))


def make_doc_history(seed, n_sites=3, n_ops=300, sync_prob=0.05, commit_prob=0.3, peers=None, unicode_=True):
    """Returns (blob, expected_json_text, expected_vv, sites) for one document."""
    rnd = random.Random(seed)
    peers = peers or [rnd.getrandbits(64) | 1 for _ in range(n_sites)]
    docs = [OracleDoc(p) for p in peers]
    hs = [(d.get_text("text"), d.get_list("list"), d.get_map("map")) for d in docs]
    for _ in range(n_ops):
        i = rnd.randrange(n_sites)
        random_edit(rnd, docs[i], *hs[i], unicode_=unicode_)
        if rnd.random() < commit_prob:
            docs[i].commit()
        if n_sites > 1 and rnd.random() < sync_prob:
            j = rnd.randrange(n_sites)
            if j != i:
                merge(docs[j], docs[i])
    for _ in range(2):
        for i in range(n_sites):
            for j in range(n_sites):
                if i != j:
                    merge(docs[i], docs[j])
    blob = docs[0].export_updates()
    fresh = OracleDoc(1)
    fresh.import_(blob)
    return blob, fresh.json_text(), fresh.oplog_vv(), docs


def c1_two_peer_list(seed=1, n_each=1000):
    """BASELINE config C1: 2 peers x n_each List inserts of I64 at random positions, one change per 10 ops;
    each side imports the other's updates.  Returns (blob_all, json_text)."""
    rnd = random.Random(seed)
    a, b = OracleDoc(1), OracleDoc(2)
    la, lb = a.get_list("list"), b.get_list("list")
    for k in range(n_each):
        a.list_insert(la, rnd.randint(0, a.seq_len(la)), rnd.randint(-10**6, 10**6))
        b.list_insert(lb, rnd.randint(0, b.seq_len(lb)), rnd.randint(-10**6, 10**6))
        if k % 10 == 9:
            a.commit(); b.commit()
    merge(a, b)
    merge(b, a)
    assert a.json_text() == b.json_text()
    return a.export_updates(), a.json_text()


def random_tree_edit(rnd, d, tree, p_create=0.35, p_delete=0.08, p_meta=0.12):
    """One random movable-tree action (handler/tree.rs): create under a random alive node or the root, move to a
    random parent / index (cycles are rejected locally, concurrent ones are resolved by the merge), delete,
    or a write into a node's meta map."""
    nodes = d.tree_nodes(tree)
    r = rnd.random()
    if not nodes or r < p_create:
        parent = rnd.choice(nodes) if nodes and rnd.random() < 0.8 else None
        try:
            d.tree_create(tree, parent, -1 if rnd.random() < 0.5 else 0)
        except IndexError:
            pass
    elif r < p_create + p_delete:
        d.tree_delete(tree, rnd.choice(nodes))
    elif r < p_create + p_delete + p_meta:
        d.map_set(d.tree_meta(rnd.choice(nodes)), "k%d" % rnd.randrange(4), rnd.randint(0, 99))
    else:
        t = rnd.choice(nodes)
        parent = rnd.choice(nodes) if rnd.random() < 0.85 else None
        try:
            d.tree_move(tree, t, parent, -1 if rnd.random() < 0.6 else 0)
        except IndexError:
            pass


def make_tree_history(seed, n_sites=3, n_base=40, n_ops=120, sync_prob=0.04, commit_prob=0.3, mixed=False):
    """C5-shaped history: peer 0 builds a base tree of n_base nodes, everybody syncs, then the sites issue
    concurrent random tree actions (moves that form cycles across sites included).  Returns
    (blob, expected_json_text, expected_vv, sites)."""
    rnd = random.Random(seed)
    peers = [rnd.getrandbits(64) | 1 for _ in range(n_sites)]
    docs = [OracleDoc(p) for p in peers]
    trees = [d.get_tree("tree") for d in docs]
    hs = [(d.get_text("text"), d.get_list("list"), d.get_map("map")) for d in docs] if mixed else None
    for _ in range(n_base):
        random_tree_edit(rnd, docs[0], trees[0], p_create=1.0)
        if rnd.random() < commit_prob:
            docs[0].commit()
    for j in range(1, n_sites):
        merge(docs[j], docs[0])
    for _ in range(n_ops):
        i = rnd.randrange(n_sites)
        if mixed and rnd.random() < 0.3:
            random_edit(rnd, docs[i], *hs[i])
        else:
            random_tree_edit(rnd, docs[i], trees[i], p_create=0.15)
        if rnd.random() < commit_prob:
            docs[i].commit()
        if n_sites > 1 and rnd.random() < sync_prob:
            j = rnd.randrange(n_sites)
            if j != i:
                merge(docs[j], docs[i])
    for _ in range(2):
        for i in range(n_sites):
            for j in range(n_sites):
                if i != j:
                    merge(docs[i], docs[j])
    blob = docs[0].export_updates()
    fresh = OracleDoc(1)
    fresh.import_(blob)
    return blob, fresh.json_text(), fresh.oplog_vv(), docs


def overlapping_update_blobs(seed):
    """Two blobs of one history whose changes overlap PARTIALLY: an early full export, then -- after the author kept
    editing, so that its stored change grew past that export -- an update cut from an older version.  Importing both
    makes the second arrive with a known head (OpLog::trim_the_known_part_of_change, oplog.rs:181-196).
    Returns (blob_early, blob_late, n_partial_overlaps)."""
    rnd = random.Random(seed)
    a, b = OracleDoc(100), OracleDoc(101)
    ha = (a.get_text("text"), a.get_list("list"), a.get_map("map"))
    hb = (b.get_text("text"), b.get_list("list"), b.get_map("map"))
    for _ in range(30):
        random_edit(rnd, a, *ha)
        random_edit(rnd, b, *hb)
        if rnd.random() < 0.3:
            a.commit(); b.commit()
    merge(a, b); merge(b, a)
    for _ in range(25):
        random_edit(rnd, a, *ha, children=0)
        if rnd.random() < 0.3:
            a.commit()
    a.commit()
    e1, vv1 = a.export_updates(), a.oplog_vv()
    for _ in range(25):
        random_edit(rnd, a, *ha, children=0)
        if rnd.random() < 0.3:
            a.commit()
    a.commit()
    e2 = a.export_updates({p: max(0, c - rnd.randint(1, 15)) for p, c in vv1.items()})
    n = 0
    for bl in oracle.decode_dump(e2)["blocks"]:
        for ch in bl["changes"]:
            end = ch["ops"][-1]["counter"] + ch["ops"][-1]["len"]
            if ch["counter"] < vv1.get(int(ch["peer"]), 0) < end:
                n += 1
    return e1, e2, n


def import_batch_order(blobs):
    """LoroDoc::import_batch imports its blobs sorted by number of changes, descending, stably (loro.rs:1194-1202)."""
    def n_changes(blob):
        return sum(len(bl["changes"]) for bl in oracle.decode_dump(blob)["blocks"])
    return sorted(blobs, key=lambda x: -n_changes(x))


def pending_only_blob():
    """A document whose one change depends on a change the blob does not carry: nothing of it is applied."""
    a = OracleDoc(5)
    a.text_insert(a.get_text("t"), 0, "abc")
    a.commit()
    vv = a.oplog_vv()
    a.text_insert(a.get_text("t"), 3, "def")
    return a.export_updates(vv)


def map_only_blob():
    a = OracleDoc(6)
    m = a.get_map("map")
    a.map_set(m, "k", 1)
    a.map_set(m, "s", "v")
    return a.export_updates()


def bad_checksum(blob):
    return blob[:30] + bytes([blob[30] ^ 1]) + blob[31:]


def skipped_kinds(blob):
    """documents the list integration kernel skips: `blob` with a bad checksum, a pending-only, a map-only and an empty
    document"""
    return [bad_checksum(blob), pending_only_blob(), map_only_blob(), OracleDoc(8).export_updates()]
