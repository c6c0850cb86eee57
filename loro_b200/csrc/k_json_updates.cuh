// loro_b200 -- the changes between two versions as Loro JSON updates (LoroDoc::export_json_updates).
//
// Replaces (reference, relative to crates/loro-internal/src):
//   loro.rs:715-751 export_json_updates, encoding/json_schema.rs:31-45 (refine_vv), :47-80 (export_json),
//   :144-169 (init_encode: Change::slice at both ends, stable sort by lamport), :270-548 (encode_change and the peer
//   register), :817-1240 (the `json` module: serde field order, internally tagged contents, ids as "counter@peer"),
//   oplog/loro_dag.rs:1036-1065 (vv_to_frontiers for start_version), change.rs:203-258 (Change::slice),
//   list_op.rs:603-658 (Op::slice), outdated_encode_reordered.rs:318-352 (create / move / delete of a tree op).
//
// The JSON lists the document's STORED changes (iter_changes_peer_by_peer walks the change store): k_jx_store rebuilds
// the import store with k_exp_store's walk (xstore_walk) and lists each stored change once in the fc_* tables, per peer
// slot.  k_jx_order (a thread per request) then orders the stored changes that overlap [start, end) by lamport -- a P-way
// merge of the per-peer lists, ties by ascending peer id (the reference leaves them in FxHashMap order) -- lists them and
// registers the peers in first-use order.  The text is printed a thread per output change: k_jx_changes counts each
// change's bytes (cutting it to [start, end) with the export's xentry_slice, whose end cut the op gather honours), the
// host scans the sizes and places every request, and k_jx_changes writes each change while k_jx_envelope writes each
// request's head and tail, one chunk of requests at a time.
#pragma once
#include "k_export.cuh"
#include "k_resolve.cuh"
#include "k_state.cuh"

#define JX_NO_PEER_COMPRESSION 1u   // LB_JSON_NO_PEER_COMPRESSION
#define JX_NONE 0xFFFFFFFFu
#define JX_UNSUPPORTED (~0ull)      // JxReq::len of a document the export phase does not cover

struct JxReq {       // one request as the host lays it out
    u32 doc;
    u32 flags;       // JX_NO_PEER_COMPRESSION
    u64 slot0;       // first of the request's P entries in the per-request scratch (start, end, register, cursors)
    u64 ch0;         // first of its slots in the output-change list (as many as its document has stored changes)
    u64 c0;          // first of its output changes in the compacted list the per-change kernels run over
    u64 off;         // offset of the request's text in the output buffer
    u64 len;         // bytes of the text (JX_UNSUPPORTED: not covered)
    u32 n_out;       // output changes (k_jx_order)
    u32 n_peers;     // peers registered (k_jx_order)
    u32 pre_len;     // bytes of the envelope in front of the changes (k_jx_order)
    u32 pad;
};
// ContainerType's name as ContainerID's Display prints it
__device__ inline void put_ctype(Sink& o, u8 type) {
    const char* names[6] = {"Map", "List", "Text", "Tree", "MovableList", "Counter"};
    o.puts_(type < 6 ? names[type] : "Unknown");
}
// ContainerID's Display (loro-common/src/lib.rs:480-500) without the quotes; put_peer(p) prints the creator of a normal
// container from its doc peer index (the JSON writer prints a register index or the id, k_attr.cuh the id)
template <class PutPeer>
__device__ __forceinline__ void put_cid_to(Sink& o, const BatchTables& t, const DocInfo& di, u32 cidx, PutPeer put_peer) {
    const DocContainer& dc = t.dcont[di.cid0 + cidx];
    if (dc.is_root) { o.puts_("cid:root-"); o.put_escaped(t.bytes + dc.name_off, dc.name_len); }
    else { o.puts_("cid:"); o.put_i64(dc.counter); o.put('@'); put_peer(dc.key_or_peer); }
    o.put(':');
    put_ctype(o, dc.type);
}

struct JxScratch {   // per request and document peer slot
    i32* start;      // refined start_vv / end_vv (json_schema.rs:31-45: clamped to the oplog vv, 0 when absent)
    i32* end;
    u32* reg;        // register index of the peer (JX_NONE: not yet used)
    u32* ord;        // the registered peers in register order
    u32* cur;        // merge cursor: next stored change of the peer (index relative to the peer's first)
};

// thread per requested document: the import store (xstore_walk), its changes listed peer by peer in slot order in fc_*;
// pf0 / pfn[peer slot] = first stored change of the peer (relative to the document's first) and how many it has
__global__ void k_jx_store(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t,
                           u32* __restrict__ pf0, u32* __restrict__ pfn) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs || !t.x_req[d]) return;
    const DocInfo& di = docs[d];
    XDoc x = t.xdoc[d];
    if (di.code != DOC_OK || (x.flags & 1)) return;
    const u64 w0 = di.ch0 + t.ch_seg0[di.ch0];
    u64 w = w0;
    for (u32 p = 0; p < di.P; p++) {
        pf0[di.peer0 + p] = (u32)(w - w0);
        xstore_walk(t, di, t.dpeer[di.peer0 + p], [] { return true; }, [&](const XEntry& e) {
            t.fc_src[w] = e.src; t.fc_pos[w] = e.pos; t.fc_r0[w] = e.r0; t.fc_from[w] = e.from; t.fc_atoms[w] = e.atoms;
            t.fc_nrows[w] = e.nrows; t.fc_skip[w] = e.skip;
            w++;
        });
        pfn[di.peer0 + p] = (u32)(w - w0) - pf0[di.peer0 + p];
    }
    x.n_fc = (u32)(w - w0);
    t.xdoc[d] = x;
}

// ---------------------------------------------------------------------------------------------- one request
struct JxWriter {
    const BatchTables& t;
    const DocInfo& di;
    JxReq& rq;
    const JxScratch& s;
    Sink& o;
    const u32* pf0;
    const u32* pfn;
    u64 fc_base;
    bool compress;

    __device__ u32 reg(u32 p) {   // ValueRegister::register (k_jx_order assigns; the text only reads)
        u32& r = s.reg[rq.slot0 + p];
        if (r == JX_NONE) { r = rq.n_peers; s.ord[rq.slot0 + rq.n_peers] = p; rq.n_peers++; }
        return r;
    }
    __device__ void put_peer(u32 p) { if (compress) o.put_u64(s.reg[rq.slot0 + p]); else o.put_u64(t.dpeer[di.peer0 + p].id); }
    __device__ void put_id(u32 p, i64 ctr) { o.put('"'); o.put_i64(ctr); o.put('@'); put_peer(p); o.put('"'); }
    __device__ void put_type(u8 type) { put_ctype(o, type); }
    __device__ void put_cid(u32 cidx) { put_cid_to(o, t, di, cidx, [&](u32 p) { put_peer(p); }); }

    // a LoroValue at c (kind byte + content), serde_json text (loro-common/src/value.rs:692-711): object keys ascending,
    // the later of two equal keys wins, a container is "🦜:" + its id, which is (peer, ctr) of the atom that created it.
    // Nested lists and maps go on an explicit stack of LB_MAX_NESTING levels, as deep as the decoder admits (so it never
    // fills, and a value is never cut short): the stack a recursive walk needs
    // cannot be sized at compile time.  A map level prints its keys by selection, O(entries^2) per level, which is cheap
    // for the small nested values documents carry.  k_state.cuh prints the same byte format, but as part of its
    // container frame machine (a child container there is expanded, here it is an id), so the two walkers stay apart.
    struct VLevel { const u8* body; const u8* after; u32 n, left, last; bool map; };
    __device__ void value(Cur& c, const BlockInfo& blk, u32 peer, i32 ctr) {
        VLevel st[LB_MAX_NESTING];
        int sp = 0;
        while (true) {
            const u8 kind = c.get();
            switch (kind) {
                case 0: o.puts_("null"); break;
                case 1: o.puts_("true"); break;
                case 2: o.puts_("false"); break;
                case 3: o.put_i64(c.sleb()); break;
                case 4: {
                    u64 bits = 0;
                    for (int i = 0; i < 8; i++) bits = (bits << 8) | c.get();
                    char buf[32];
                    int n = f64_format(bits, buf);
                    for (int i = 0; i < n; i++) o.put((u8)buf[i]);
                    break;
                }
                case 5: case 6: {
                    u64 n = c.varint();
                    if (n > c.left()) n = c.left();
                    if (kind == 5) { o.put('"'); o.put_escaped(c.p, n); o.put('"'); }
                    else { o.put('['); for (u64 i = 0; i < n; i++) { if (i) o.put(','); o.put_u64(c.p[i]); } o.put(']'); }
                    c.skip(n);
                    break;
                }
                case 7: case 8: {
                    const u32 n = (u32)c.varint();
                    if (sp == LB_MAX_NESTING) { c.err = 1; break; }
                    VLevel& l = st[sp++];
                    l.map = kind == 8; l.n = l.left = n; l.last = JX_NONE; l.body = c.p;
                    if (l.map) for (u32 i = 0; i < n && !c.err; i++) { (void)c.varint(); u8 k = c.get(); skip_loro_value_content(c, k, nullptr); }
                    l.after = c.p;
                    o.put(l.map ? '{' : '[');
                    break;
                }
                case 9: {
                    const u8 type = c.get();
                    o.puts_("\"🦜:cid:");
                    o.put_i64(ctr);
                    o.put('@');
                    put_peer(peer);
                    o.put(':');
                    put_type(type);
                    o.put('"');
                    break;
                }
                default: o.puts_("null"); c.err = 1;
            }
            // the next value to print: the next item of the innermost open list, or the next key of the innermost map
            bool more = false;
            while (sp && !more && !c.err) {
                VLevel& l = st[sp - 1];
                if (!l.map) {
                    if (!l.left) { o.put(']'); sp--; continue; }
                    if (l.left < l.n) o.put(',');
                    l.left--;
                    more = true;
                    continue;
                }
                Cur e(l.body, (size_t)(l.after - l.body));
                u32 best = JX_NONE;
                const u8* best_val = nullptr;
                for (u32 i = 0; i < l.n && !e.err; i++) {
                    u32 ki = (u32)e.varint();
                    const u8* val = e.p;
                    u8 k = e.get();
                    skip_loro_value_content(e, k, nullptr);
                    if (ki >= blk.n_keys) continue;
                    if (l.last != JX_NONE && key_cmp(blk, ki, l.last) <= 0) continue;
                    if (best == JX_NONE || key_cmp(blk, ki, best) <= 0) { best = ki; best_val = val; }
                }
                if (best == JX_NONE) { o.put('}'); c.p = l.after; sp--; continue; }
                if (l.last != JX_NONE) o.put(',');
                l.last = best;
                o.put('"');
                o.put_escaped(t.bytes + t.key_off[blk.key0 + best], t.key_len[blk.key0 + best]);
                o.puts_("\":");
                c.p = best_val;
                more = true;
            }
            if (!more) return;
        }
    }
    __device__ int key_cmp(const BlockInfo& blk, u32 a, u32 b) {
        const u8* pa = t.bytes + t.key_off[blk.key0 + a];
        const u8* pb = t.bytes + t.key_off[blk.key0 + b];
        u32 la = t.key_len[blk.key0 + a], lb = t.key_len[blk.key0 + b];
        u32 n = la < lb ? la : lb;
        for (u32 i = 0; i < n; i++) if (pa[i] != pb[i]) return pa[i] < pb[i] ? -1 : 1;
        return la < lb ? -1 : (la > lb ? 1 : 0);
    }

    // the stored change k cut to [start, end) of its peer (Change::slice at both ends): false when nothing of it lies there
    __device__ bool entry(u32 p, u32 k, XEntry& E) {
        const u64 f = fc_base + pf0[di.peer0 + p] + k;
        E.src = t.fc_src[f]; E.from = t.fc_from[f]; E.pos = t.fc_pos[f]; E.r0 = t.fc_r0[f]; E.atoms = t.fc_atoms[f];
        E.nrows = t.fc_nrows[f]; E.skip = t.fc_skip[f]; E.tail = 0; E.last_valid = false;
        const i32 st = s.start[rq.slot0 + p], en = s.end[rq.slot0 + p];
        if (st >= en) return false;   // from.diff_iter(to) holds nothing of the peer
        const i32 c0 = t.ch_counter[E.src] + (i32)E.from;
        if (c0 >= en || c0 + (i32)E.atoms <= st) return false;
        xentry_slice(t, E, st, en);
        return true;
    }

    // the ops of E: f(op, cursor at its first row, atoms of that row outside the op)
    template <class F>
    __device__ void ops(const XEntry& E, F f) {
        XRows it(t, E.pos, E.r0);
        u32 left = E.nrows;
        bool first = true;
        while (left) {
            XRows at = it;
            const u32 skip = first ? E.skip : it.skip;
            first = false;
            f(xop_gather(t, di, it, left, skip, E.tail), at, skip);
        }
    }
    // the items (List) or text (Text) of an insert, `take` atoms from the cursor on: f(cursor, payload of the row
    // without its skipped atoms, its bytes, atoms to print, atoms in the payload)
    template <class F>
    __device__ void payload(XRows at, u32 skip, u32 xk, u32 take, F f) {
        while (take) {
            const u8* pp;
            u32 pn;
            xr_payload_skip(t, at.row(), xk, skip, &pp, &pn);
            const u32 avail = xr_len(t, at.row()) - skip;
            f(at, pp, pn, avail < take ? avail : take, avail);
            take -= avail < take ? avail : take;
            if (take) { at.next(); skip = at.skip; }
        }
    }

    // encode_change's register order (json_schema.rs:301-548): per op its container (normal ids), the containers among
    // its values, a delete's start id, a tree op's target and parent; then the change id; then the sorted deps
    __device__ void register_change(const XEntry& E, u32 cp) {
        ops(E, [&](const XOp& op, XRows at, u32 skip) {
            const DocContainer& dc = t.dcont[di.cid0 + op.cidx];
            if (!dc.is_root) reg(dc.key_or_peer);
            if (op.xk == XK_LIST) {
                payload(at, skip, XK_LIST, op.atoms, [&](XRows&, const u8* pp, u32 pn, u32 n, u32) {
                    Cur c(pp, pn);
                    for (u32 i = 0; i < n && !c.err; i++) { u8 k = c.get(); if (k == 9) reg(cp); skip_loro_value_content(c, k, nullptr); }
                });
            } else if (op.xk == XK_MAPSET) {
                const u8* pp;
                u32 pn;
                xr_payload(t, at.row(), XK_MAPSET, &pp, &pn);
                if (pn && pp[0] == 9) reg(cp);
            } else if (op.xk == XK_DEL) reg(op.f0);
            else if (op.xk == XK_TREE) {
                uint4 ids = t.tr_ids[op.f0];
                reg(ids.x);
                if ((ids.z & 3u) == TRP_NODE) reg(ids.z >> 2);
            }
        });
        reg(cp);
        deps(E, [&](u32 p, i32) { reg(p); });
    }
    // the deps of E ascending by (peer id, counter): a front-sliced change depends on its own previous atom
    template <class F>
    __device__ void deps(const XEntry& E, F f) {
        const u32 cp = t.ch_peer[E.src];
        if (E.from) { f(cp, t.ch_counter[E.src] + (i32)E.from - 1); return; }
        const BlockInfo& sb = t.blocks[t.ch_block[E.src]];
        const u32 nd = t.ch_ndeps[E.src];
        const bool self = t.ch_dep_self[E.src] != 0;
        u64 lp = 0; i32 lc = 0;
        bool any = false;
        for (u32 n = 0; n < nd + (self ? 1u : 0u); n++) {   // selection: the next dep above the last one
            u32 bp = JX_NONE; i32 bc = 0; u64 bid = 0;
            for (u32 k = 0; k <= nd; k++) {
                u32 p; i32 c;
                if (k == nd) { if (!self) continue; p = cp; c = t.ch_counter[E.src] - 1; }
                else { p = t.peer_map[sb.peer0 + t.dep_peer_idx[t.ch_dep0[E.src] + k]]; c = t.dep_counter[t.ch_dep0[E.src] + k]; }
                u64 id = t.dpeer[di.peer0 + p].id;
                if (any && (id < lp || (id == lp && c <= lc))) continue;
                if (bp == JX_NONE || id < bid || (id == bid && c < bc)) { bp = p; bc = c; bid = id; }
            }
            if (bp == JX_NONE) break;
            f(bp, bc);
            lp = bid; lc = bc; any = true;
        }
    }

    __device__ void put_change(const XEntry& E) {
        const u32 cp = t.ch_peer[E.src];
        const i32 c0 = t.ch_counter[E.src] + (i32)E.from;
        o.puts_("{\"id\":");
        put_id(cp, c0);
        o.puts_(",\"timestamp\":");
        o.put_i64(t.ch_ts[E.src]);
        o.puts_(",\"deps\":[");
        bool first = true;
        deps(E, [&](u32 p, i32 c) { if (!first) o.put(','); first = false; put_id(p, c); });
        o.puts_("],\"lamport\":");
        o.put_u64((u64)t.ch_lamport[E.src] + E.from);
        o.puts_(",\"msg\":");
        if (t.ch_msg_len[E.src]) { o.put('"'); o.put_escaped(t.bytes + t.ch_msg_off[E.src], t.ch_msg_len[E.src]); o.put('"'); }
        else o.puts_("null");
        o.puts_(",\"ops\":[");
        first = true;
        ops(E, [&](const XOp& op, XRows at, u32 skip) {
            if (!first) o.put(',');
            first = false;
            o.puts_("{\"container\":\"");
            put_cid(op.cidx);
            o.puts_("\",\"content\":{\"type\":");
            switch (op.xk) {
                case XK_LIST: case XK_TEXT: {
                    const bool text = op.xk == XK_TEXT;
                    o.puts_("\"insert\",\"pos\":");
                    o.put_i64(op.prop);
                    o.puts_(text ? ",\"text\":\"" : ",\"value\":[");
                    u32 i = 0;
                    payload(at, skip, op.xk, op.atoms, [&](XRows& r, const u8* pp, u32 pn, u32 n, u32 avail) {
                        if (text) { o.put_escaped(pp, text_byte_index(pp, pn, avail, n)); return; }
                        Cur c(pp, pn);
                        const BlockInfo& blk = t.blocks[t.ch_block[r.ch]];
                        for (u32 k = 0; k < n && !c.err; k++, i++) { if (i) o.put(','); value(c, blk, cp, op.ctr + (i32)i); }
                    });
                    o.puts_(text ? "\"" : "]");
                    break;
                }
                case XK_DEL: {
                    o.puts_("\"delete\",\"pos\":");
                    o.put_i64(op.prop);
                    o.puts_(",\"len\":");
                    o.put_i64(op.f2);
                    o.puts_(",\"start_id\":");
                    put_id(op.f0, (i32)op.f1);
                    break;
                }
                case XK_MAPSET: case XK_MAPDEL: {
                    o.puts_(op.xk == XK_MAPSET ? "\"insert\",\"key\":\"" : "\"delete\",\"key\":\"");
                    o.put_escaped(t.bytes + t.dkey_off[di.key0 + (u32)op.prop], t.dkey_len[di.key0 + (u32)op.prop]);
                    o.put('"');
                    if (op.xk == XK_MAPSET) {
                        const u8* pp;
                        u32 pn;
                        xr_payload(t, at.row(), XK_MAPSET, &pp, &pn);
                        o.puts_(",\"value\":");
                        Cur c(pp, pn);
                        value(c, t.blocks[t.ch_block[at.ch]], cp, op.ctr);
                    }
                    break;
                }
                case XK_TREE: {
                    const uint4 ids = t.tr_ids[op.f0];
                    const u32 pk = ids.z & 3u;
                    const bool create = ids.x == cp && (i32)ids.y == op.ctr;
                    o.puts_(pk == TRP_DELETED ? "\"delete\"" : (create ? "\"create\"" : "\"move\""));
                    o.puts_(",\"target\":");
                    put_id(ids.x, (i32)ids.y);
                    if (pk != TRP_DELETED) {
                        o.puts_(",\"parent\":");
                        if (pk == TRP_ROOT) o.puts_("null"); else put_id(ids.z >> 2, (i32)ids.w);
                        o.puts_(",\"fractional_index\":\"");
                        const u32 pos = t.tr_pos[op.f0];
                        const char* HEX = "0123456789ABCDEF";   // crates/fractional_index/src/lib.rs:195-205
                        for (u32 k = 0; k < t.pos_len[pos]; k++) {
                            u8 b = t.pos_pool[t.pos_off[pos] + k];
                            o.put((u8)HEX[b >> 4]); o.put((u8)HEX[b & 15]);
                        }
                        o.put('"');
                    }
                    break;
                }
                default: o.puts_("\"unknown\"");
            }
            o.puts_("},\"counter\":");
            o.put_i64(op.ctr);
            o.put('}');
        });
        o.puts_("]}");
    }

    // vv_to_frontiers of the refined start (loro_dag.rs:1036-1065): the last id of every peer the start holds, unless
    // the causal past of another one includes it; an object from decimal peer id to counter, peer ids ascending
    __device__ void put_start_version() {
        const u32 P = di.P;
        o.put('{');
        bool first = true;
        for (u32 rank = 0; rank < P; rank++) {
            u32 p = 0;
            while (p < P && t.dpeer[di.peer0 + p].rank != rank) p++;
            if (p == P) break;
            const i32 sp = s.start[rq.slot0 + p];
            if (sp <= 0) continue;
            bool covered = false;
            for (u32 q = 0; q < P && !covered; q++) {
                const i32 sq = s.start[rq.slot0 + q];
                if (q == p || sq <= 0) continue;
                u32 lam, ch;
                if (!lamport_of(di, t, q, sq - 1, &lam, &ch)) continue;
                covered = t.ch_vv[di.vv0 + (u64)t.ch_pos[ch] * P + p] >= sp;
            }
            if (covered) continue;
            if (!first) o.put(',');
            first = false;
            o.put('"');
            o.put_u64(t.dpeer[di.peer0 + p].id);
            o.puts_("\":");
            o.put_i64(sp - 1);
        }
        o.put('}');
    }
    __device__ void put_peers() {
        if (!compress) { o.puts_("null"); return; }
        o.put('[');
        for (u32 i = 0; i < rq.n_peers; i++) {
            if (i) o.put(',');
            o.put('"');
            o.put_u64(t.dpeer[di.peer0 + s.ord[rq.slot0 + i]].id);
            o.put('"');
        }
        o.put(']');
    }

    __device__ void put_prefix() {
        o.puts_("{\"schema_version\":1,\"start_version\":");
        put_start_version();
        o.puts_(",\"peers\":");
        put_peers();
        o.puts_(",\"changes\":[");
    }

    // the P-way merge of the per-peer lists (lamport rises along a peer's chain): och[rq.ch0 + i] = the i-th output change
    // (stored change index relative to the document's first); the peers are registered in output order
    __device__ void order(u32* och) {
        const u32 P = di.P;
        for (u32 p = 0; p < P; p++) { s.cur[rq.slot0 + p] = 0; s.reg[rq.slot0 + p] = JX_NONE; }
        rq.n_peers = 0;
        u32 n = 0;
        while (true) {
            u32 best = JX_NONE;
            u64 best_key = 0;
            for (u32 p = 0; p < P; p++) {   // each peer's first stored change that overlaps [start, end)
                const i32 st = s.start[rq.slot0 + p], en = s.end[rq.slot0 + p];
                u32& k = s.cur[rq.slot0 + p];
                const u32 np = st < en ? pfn[di.peer0 + p] : 0;
                u64 f = 0;
                i32 c0 = 0;
                for (; k < np; k++) {
                    f = fc_base + pf0[di.peer0 + p] + k;
                    c0 = t.ch_counter[t.fc_src[f]] + (i32)t.fc_from[f];
                    if (c0 >= en) { k = np; break; }
                    if (c0 + (i32)t.fc_atoms[f] > st) break;
                }
                if (k >= np) continue;
                const u32 cut = st > c0 ? (u32)(st - c0) : 0u;   // Change::slice moves the lamport by the cut
                const u64 key = ((u64)(t.ch_lamport[t.fc_src[f]] + t.fc_from[f] + cut) << 32) | t.dpeer[di.peer0 + p].rank;
                if (best == JX_NONE || key < best_key) { best = p; best_key = key; }
            }
            if (best == JX_NONE) break;
            const u32 k = s.cur[rq.slot0 + best]++;
            XEntry E;
            entry(best, k, E);
            if (compress) register_change(E, t.ch_peer[E.src]);
            och[rq.ch0 + n++] = pf0[di.peer0 + best] + k;
        }
        rq.n_out = n;
    }
    // output change `rank` of the request: its stored change `rel`, printed with the comma that separates it
    __device__ void change_text(u32 rel, u32 rank) {
        const u32 p = t.ch_peer[t.fc_src[fc_base + rel]];
        XEntry E;
        entry(p, rel - pf0[di.peer0 + p], E);
        if (rank) o.put(',');
        put_change(E);
    }
};

__device__ __forceinline__ JxWriter jx_writer(const DocInfo* docs, const BatchTables& t, JxReq& rq, const JxScratch& s,
                                              Sink& o, const u32* pf0, const u32* pfn) {
    const DocInfo& di = docs[rq.doc];
    return JxWriter{t, di, rq, s, o, pf0, pfn, di.ch0 + t.ch_seg0[di.ch0], !(rq.flags & JX_NO_PEER_COMPRESSION)};
}
__device__ __forceinline__ Sink jx_sink(u8* dst) { Sink o; o.dst = dst; o.n = 0; o.flags = 0; o.wr = true; return o; }

// thread per request: order its changes, register its peers, size its envelope
__global__ void k_jx_order(const DocInfo* __restrict__ docs, const __grid_constant__ BatchTables t, JxReq* __restrict__ reqs,
                           u32 n_reqs, JxScratch s, const u32* __restrict__ pf0, const u32* __restrict__ pfn, u32* __restrict__ och) {
    u32 r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reqs) return;
    JxReq& rq = reqs[r];
    if (t.xdoc[rq.doc].flags & 1) { rq.len = JX_UNSUPPORTED; rq.n_out = 0; return; }
    Sink o = jx_sink(nullptr);
    JxWriter w = jx_writer(docs, t, rq, s, o, pf0, pfn);
    w.order(och);
    w.put_prefix();
    rq.pre_len = (u32)o.n;
}

// thread per output change of [k_lo, k_hi) (compacted numbering; oreq = its request).  len != null: count its bytes into
// len[k]; otherwise write it at off[k] - out_base
__global__ void k_jx_changes(const DocInfo* __restrict__ docs, const __grid_constant__ BatchTables t, JxReq* __restrict__ reqs,
                             JxScratch s, const u32* __restrict__ pf0, const u32* __restrict__ pfn, const u32* __restrict__ och,
                             const u32* __restrict__ oreq, u64 k_lo, u64 k_hi, u32* __restrict__ len,
                             const u64* __restrict__ off, u8* __restrict__ out, u64 out_base) {
    const u64 k = k_lo + (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= k_hi) return;
    JxReq& rq = reqs[oreq[k]];
    const u32 rank = (u32)(k - rq.c0);
    Sink o = jx_sink(len ? nullptr : out + (off[k] - out_base));
    JxWriter w = jx_writer(docs, t, rq, s, o, pf0, pfn);
    w.change_text(och[rq.ch0 + rank], rank);
    if (len) len[k] = (u32)o.n;
}

// thread per request of [r_lo, r_hi): the envelope around its changes
__global__ void k_jx_envelope(const DocInfo* __restrict__ docs, const __grid_constant__ BatchTables t, JxReq* __restrict__ reqs,
                              u32 r_lo, u32 r_hi, JxScratch s, const u32* __restrict__ pf0, const u32* __restrict__ pfn,
                              u8* __restrict__ out, u64 out_base) {
    const u32 r = r_lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= r_hi) return;
    JxReq& rq = reqs[r];
    if (rq.len == JX_UNSUPPORTED) return;
    Sink o = jx_sink(out + (rq.off - out_base));
    JxWriter w = jx_writer(docs, t, rq, s, o, pf0, pfn);
    w.put_prefix();
    out[rq.off - out_base + rq.len - 2] = ']';
    out[rq.off - out_base + rq.len - 1] = '}';
}
