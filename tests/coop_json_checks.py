"""Documents whose List and Text containers have many visible runs, built to hit the edges of the state JSON writer that
prints such a container 32 pieces at a time (one list element or one text run per lane): runs that straddle the
32-element windows, runs that start inside their op, pieces exactly at, under and over the 32-byte staging slot,
escaped text bytes at run edges, a nested value after several windows, containers of 63, 64 and 65 runs, each under
root names of 1 to 4 bytes so that the windows start and end at every offset within a word.  Shared by
test_coop_json_emu.py and test_coop_json_gpu.py; every document's JSON is compared with the oracle's byte for byte."""
from oracle import OracleDoc

from .engine_checks import check_batch_against_oracle

ROOTS = ["a", "ab", "abc", "abcd"]


def _doc(build, root):
    d = OracleDoc(7)
    build(d, root)
    d.commit()
    return d.export_updates()


def _list(groups, deletes=()):
    """one run per group: each group is inserted at the front in one op (the list holds them in reverse order);
    deletes (pos, n) then apply to the final list"""
    def build(d, root):
        c = d.get_list(root)
        for g in groups:
            d.list_insert(c, 0, *g)
        for pos, n in deletes:
            d.delete(c, pos, n)
    return build


def _text(pieces, deletes=()):
    def build(d, root):
        c = d.get_text(root)
        for s in pieces:
            d.text_insert(c, 0, s)
        for pos, n in deletes:
            d.delete(c, pos, n)
    return build


def _value(i):
    k = i % 7
    if k == 0:
        return (i * 7919) % 2000001 - 1000000
    if k == 1:
        return "ab\"\\c"[: i % 6]
    if k == 2:
        return i * 0.25 - 3.0
    if k == 3:
        return None
    if k == 4:
        return i % 2 == 0
    if k == 5:
        return -(2 ** 63) + i
    return "x" * (i % 9)


def straddle_groups():
    """run lengths 1..9, 31, 32, 33, 40: every window boundary falls inside some run and at some run's edge"""
    lens = [1, 2, 3, 31, 4, 5, 32, 6, 7, 33, 8, 9, 40] * 6
    out, i = [], 0
    for n in lens:
        out.append([_value(i + j) for j in range(n)])
        i += n
    return out


def split_runs():
    """70 ops of 5 elements; in the final list each op loses its middle element (two runs, the second at offset 3)
    and every other op also its first (a run at offset 1)"""
    groups = [[_value(5 * g + j) for j in range(5)] for g in range(70)]
    deletes = []
    for q in reversed(range(70)):   # q-th op of the final list starts at 5q; delete from the back
        deletes.append((5 * q + 2, 1))
        if q % 2:
            deletes.append((5 * q, 1))
    return groups, deletes


def slot_values():
    """printed lengths around the 32-byte slot (with the comma every element but the first has)"""
    esc = "\x01"
    vals = ["s" * 27, "s" * 28, "s" * 29, "s" * 30, "s" * 31, "\"" * 14, "\"" * 15, "\\" * 15, esc * 4 + "ab", esc * 5,
            esc * 5 + "x", "q" * 100, esc * 40, -(2 ** 63), 1.7976931348623157e308, -2.2250738585072014e-308, "é語🦜" * 3,
            "é語🦜" * 4, 7, ""]
    out = []
    for i in range(72):
        n = 1 + i % 3
        out.append([vals[(i + j) % len(vals)] for j in range(n)])
    return out


def text_pieces(n, seed=0):
    """n pieces of 1..40 characters with quotes, backslashes, control bytes and multi-byte characters at their edges"""
    edge = ["\"", "\\", "\n", "\x01", "é", "語", "🦜", "\x1f", "a"]
    out = []
    for i in range(n):
        k = (i * 7 + seed) % 40 + 1
        body = "".join("abc d"[(i + j) % 5] for j in range(max(0, k - 2)))
        s = edge[i % len(edge)] + body + edge[(i * 5 + 3) % len(edge)]
        if i % 11 == 0:
            s = "\"" * 17   # 34 escaped bytes: past the slot
        if i % 13 == 0:
            s = "\\" * 16   # exactly the slot
        out.append(s)
    return out


def cases():
    sg = straddle_groups()
    groups, deletes = split_runs()
    sv = slot_values()
    nested = [[1, [2, "x"]]] + [[_value(i), _value(i + 1)] for i in range(80)]   # the nested value prints last
    tp = text_pieces(90)
    tdel = []
    pos = sum(len(s) for s in tp)
    for s in tp:   # the final text holds the pieces in reverse order: the first piece inserted ends it
        pos -= len(s)
        if len(s) > 2 and (pos % 3 == 0):
            tdel.append((pos + 1, 1))   # a run that starts inside its op after the text of its first character
    tdel.sort(reverse=True)
    builds = [
        ("list_straddle", _list(sg)),
        ("list_split_runs", _list(groups, deletes)),
        ("list_slot_edges", _list(sv)),
        ("list_nested_after_windows", _list(nested)),
        ("text_escapes", _text(tp)),
        ("text_split_runs", _text(tp, tdel)),
    ]
    for n in (63, 64, 65):
        builds.append((f"list_{n}_runs", _list([[_value(i), _value(i + 3)] for i in range(n)])))
        builds.append((f"text_{n}_runs", _text(text_pieces(n, seed=n))))
    out = []
    for name, build in builds:
        for root in ROOTS:
            out.append((f"{name}/{root}", _doc(build, root)))
    return out


def check(lib_path=None):
    cs = cases()
    check_batch_against_oracle([b for _, b in cs], lib_path=lib_path)
