"""Pins the UpdatesInRange reference (tests/range_export_ref.cpp) to the reference's behaviour: its own
loro_import_batch_status test, the identities with all_updates / updates(from) / checkout, and the rules of
export_blocks_in_range (normalised and negative spans, request order deciding block boundaries, the refused cases)."""
import json
import random

import pytest

from oracle import OracleDoc
from tests import workloads
from tests.checkout_checks import json_at
from tests.range_export_checks import BATCH_STATUS_SPANS, Refused, export_in_range, hello_docs, till_spans


def n_blocks(blob):
    """blocks of a FastUpdates body: ULEB length + block, after the 22-byte header"""
    i, n = 22, 0
    while i < len(blob):
        ln, s = 0, 0
        while True:
            b = blob[i]
            i += 1
            ln |= (b & 0x7F) << s
            s += 7
            if b < 0x80:
                break
        i += ln
        n += 1
    return n


def roots(text):
    """deep value without the empty root containers (a site lists the roots it opened, an importer those with ops)"""
    return {k: v for k, v in json.loads(text).items() if v not in ({}, [], "")}


def history(seed):
    blob = workloads.make_doc_history(seed, n_sites=3, n_ops=160)[0]
    d = OracleDoc(1)
    d.import_(blob)
    return d


def test_loro_import_batch_status():
    """crates/loro/tests/loro_rust_test.rs:2411-2460"""
    refs = hello_docs()
    b11, b12, b13, b21, b22, b23 = (export_in_range(refs[s[0][0] - 1], s) for s in BATCH_STATUS_SPANS)
    new = OracleDoc(9)
    st = new.import_batch([b11, b13, b21, b23])
    assert st["success"] == {1: (0, 5), 2: (0, 5)} and st["pending"] == {1: (6, 12), 2: (6, 12)}
    st = new.import_batch([b12, b22])
    assert st["success"] == {1: (5, 12), 2: (5, 12)} and not st["pending"]
    assert new.json_text() == b'{"text":"Hello world!Hello world!"}'


@pytest.mark.parametrize("seed", range(3))
def test_whole_and_from_spans(seed):
    d = history(7000 + seed)
    vv = d.oplog_vv()
    assert export_in_range(d, till_spans(vv)) == d.export_updates()
    rnd = random.Random(seed)
    frm = {p: rnd.randint(0, c) for p, c in vv.items()}
    assert export_in_range(d, [(p, frm[p], c) for p, c in vv.items()]) == d.export_updates(frm)


@pytest.mark.parametrize("seed", range(3))
def test_updates_till_a_causally_closed_version_is_the_checkout(seed):
    """a site's oplog vv during the run is causally closed: importing updates_till(vv) gives what checkout gives there"""
    rnd = random.Random(seed)
    docs = [OracleDoc(rnd.getrandbits(64) | 1) for _ in range(3)]
    hs = [(x.get_text("text"), x.get_list("list"), x.get_map("map")) for x in docs]
    marks = []
    for step in range(150):
        i = rnd.randrange(3)
        workloads.random_edit(rnd, docs[i], *hs[i])
        if rnd.random() < 0.3:
            docs[i].commit()
        if rnd.random() < 0.1:
            j = rnd.randrange(3)
            if j != i:
                workloads.merge(docs[j], docs[i])
        if rnd.random() < 0.1:
            docs[i].commit()
            marks.append((docs[i].oplog_vv(), docs[i].frontiers(), docs[i].json_text()))
    for i in range(3):
        for j in range(3):
            if i != j:
                workloads.merge(docs[i], docs[j])
    full = docs[0]
    assert marks
    for vv, frontiers, text in marks:
        fresh = OracleDoc(2)
        fresh.import_(export_in_range(full, till_spans(vv)))
        assert roots(fresh.json_text()) == roots(text) == roots(json_at(full, frontiers))


def test_normalised_and_negative_spans():
    d = history(7100)
    p, c = min(d.oplog_vv().items())
    assert c > 8
    assert export_in_range(d, [(p, 6, 2)]) == export_in_range(d, [(p, 3, 7)])       # covers end+1 .. start+1
    empty = OracleDoc(1).export_updates()
    assert export_in_range(d, [(p, -2, 5)]) == empty                                 # starts below 0: nothing
    assert export_in_range(d, [(p, 4, -3)]) == empty                                 # normalises to -2 .. 5
    assert export_in_range(d, [(p, 4, 4)]) == empty
    assert export_in_range(d, [(0xFEEDFACE, 0, 4)]) == empty
    assert export_in_range(d, [(p, 2, c + 50)]) == export_in_range(d, [(p, 2, c)])   # cut at the vv
    assert export_in_range(d, [(p, c, c + 5)]) == empty


def test_request_order_decides_block_boundaries():
    d = history(7200)
    p, c = min(d.oplog_vv().items())
    a = c // 2
    one = export_in_range(d, [(p, 0, c)])
    assert export_in_range(d, [(p, 0, a), (p, a, c)]) == one                          # continues the block
    two = export_in_range(d, [(p, a, c), (p, 0, a)])                                  # the higher span first
    assert n_blocks(one) == 1 and n_blocks(two) == 2 and two != one
    fresh = OracleDoc(3)
    fresh.import_(two)
    want = OracleDoc(3)
    want.import_(one)
    assert fresh.json_text() == want.json_text()


def test_refused_span_sets():
    d = history(7300)
    p, c = min(d.oplog_vv().items())
    for spans in ([(p, 0, 2), (p, 4, c)],          # a gap above an earlier-listed span: counter should be continuous
                  [(p, 0, 5), (p, 3, c)],          # overlap
                  [(p, 3, 5), (p, 3, 5)],          # the same span twice
                  [(p, 0, 3), (p, 5, 8), (p, 3, 5)]):
        with pytest.raises(Refused):
            export_in_range(d, spans)
    export_in_range(d, [(p, 5, 8), (p, 0, 3), (p, 3, 5)])   # every span finds the block below it ending at its start
