// loro_b200 -- phase 6b: who wrote each part of a document's state (attribution), as one canonical JSON object.
//
// Answers, for the whole document at the version its state was built at (reference, crates/loro/src/lib.rs):
//   :1906 LoroList::get_id_at / :2644 LoroText::get_editor_at_unicode_pos   the ids of the visible elements
//     (state/list_state.rs:326, richtext_state id_at): the visible runs phase 5 left in out_row / out_off / out_len
//   :2117 LoroMap::get_last_editor (state/map_state.rs:240)   the LWW winner of every key, deletes included: map_row
//   :3046 LoroTree::get_last_move_id (state/tree_state.rs:1034)   the last effective move of every node the tree state
//     holds, alive or deleted (creation counts as a move): tn_move
// Format (INTEGRATION.md):
//   {"peers":["<id>",...],"containers":{"<cid>":<entry>,...}}
//   Text / List  [[p,counter,len],...]        visible elements in document order, maximal runs of one peer with
//                                             consecutive counters (unicode scalar values for Text)
//   Map          {"<key>":[p,lamport,present],...}   keys ascending
//   Tree         {"<counter>@<peer>":[p,counter,alive],...}   nodes by (peer, counter)
// p indexes `peers` (the oplog vv's peers, ascending).  Containers: roots by (name bytes, type), then normal ones by
// (peer, counter); only those with an entry.
//
// Shape: a warp per document, two passes (count, write) like k_json.  The sequential frame (peers, container ids) is
// counted by every lane and written by lane 0; the entries of one container are items printed a lane each: a lane's
// item length, a warp prefix sum for its offset, then the write.  Text / List runs are merged on the fly: a lane starts
// a new item unless its (peer, first counter) continues the (peer, end) of the run before it (the lane below, or the
// last lane of the previous chunk of 32), and the lane holding the last run of an item prints it.  Map keys are ranked
// once per document (warp bitonic sort into a scratch table, pass 0) and every map of the document walks that order;
// containers are sorted the same way.  Peer ids are formatted once per document into shared memory.
#pragma once
#include "k_json_updates.cuh"

#define ATTR_SMEM_PEERS 32   // documents with more peers format ids and look ranks up from the global tables
struct AttrSmem {
    u8 txt[ATTR_SMEM_PEERS][20];
    u8 len[ATTR_SMEM_PEERS];
    u8 vix[ATTR_SMEM_PEERS];   // doc peer slot -> index into "peers"
    u8 ord[ATTR_SMEM_PEERS];   // rank -> doc peer slot
};

struct AttrWriter {
    const BatchTables& t;
    const DocInfo& di;
    Sink& out;
    const int lane;
    AttrSmem* sm;
    const bool fast;   // di.P <= ATTR_SMEM_PEERS
    u32* cord;         // the document's containers in output order (di.cid0 based)
    u32* kord;         // its keys in ascending byte order (di.key0 based)

    __device__ AttrWriter(const BatchTables& t_, const DocInfo& di_, Sink& o, int lane_, AttrSmem* sm_, u32* cord_, u32* kord_)
        : t(t_), di(di_), out(o), lane(lane_), sm(sm_), fast(di_.P <= ATTR_SMEM_PEERS), cord(cord_ + di_.cid0),
          kord(kord_ + di_.key0) {}

    __device__ const DocPeer& peer(u32 q) const { return t.dpeer[di.peer0 + q]; }
    // index of doc peer slot q in "peers": the peers of the oplog vv (end_counter > 0) with a smaller id
    __device__ u32 vix_slow(u32 q) const {
        u32 n = 0;
        const u64 id = peer(q).id;
        for (u32 r = 0; r < di.P; r++) n += peer(r).end_counter > 0 && peer(r).id < id;
        return n;
    }
    __device__ u32 vix(u32 q) const { return fast ? sm->vix[q] : vix_slow(q); }
    __device__ u32 slot_of_rank(u32 r) const {
        if (fast) return sm->ord[r];
        for (u32 q = 0; q < di.P; q++) if (peer(q).rank == r) return q;
        return 0;
    }
    __device__ u32 id_len(u32 q) const { return fast ? sm->len[q] : dec_digits(peer(q).id); }
    __device__ void put_id(Sink& o, u32 q) const {
        if (fast) for (u32 k = 0; k < sm->len[q]; k++) o.put(sm->txt[q][k]);
        else o.put_u64(peer(q).id);
    }

    // the per-document peer table (lane q formats peer q)
    __device__ void load_peers() {
        if (!fast) return;
        __syncwarp();
        if ((u32)lane < di.P) {
            const DocPeer& dp = peer(lane);
            char tmp[20];
            int k = 0;
            u64 v = dp.id;
            do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
            sm->len[lane] = (u8)k;
            for (int i = 0; i < k; i++) sm->txt[lane][i] = (u8)tmp[k - 1 - i];
            sm->vix[lane] = (u8)vix_slow(lane);
            sm->ord[dp.rank < ATTR_SMEM_PEERS ? dp.rank : 0] = (u8)lane;
        }
        __syncwarp();
    }

    __device__ int cmp_bytes(const u8* a, u32 al, const u8* b, u32 bl) const {
        u32 n = al < bl ? al : bl;
        for (u32 i = 0; i < n; i++)
            if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
        return al < bl ? -1 : (al > bl ? 1 : 0);
    }
    // pass 0: the container and key orders, kept in the scratch tables for pass 1
    __device__ void sort_tables() {
        for (u32 c = lane; c < di.C; c += 32) cord[c] = c;
        for (u32 k = lane; k < di.K; k += 32) kord[k] = k;
        __syncwarp();
        warp_sort_vals(cord, di.C, lane, [&](u32 a, u32 b) {
            const DocContainer& x = t.dcont[di.cid0 + a];
            const DocContainer& y = t.dcont[di.cid0 + b];
            if (x.is_root != y.is_root) return x.is_root > y.is_root;
            if (x.is_root) {
                int c = cmp_bytes(t.bytes + x.name_off, x.name_len, t.bytes + y.name_off, y.name_len);
                return c ? c < 0 : x.type < y.type;
            }
            if (x.peer != y.peer) return x.peer < y.peer;
            return x.counter != y.counter ? x.counter < y.counter : x.type < y.type;
        });
        warp_sort_vals(kord, di.K, lane, [&](u32 a, u32 b) {
            return cmp_bytes(t.bytes + t.dkey_off[di.key0 + a], t.dkey_len[di.key0 + a],
                             t.bytes + t.dkey_off[di.key0 + b], t.dkey_len[di.key0 + b]) < 0;
        });
    }

    // one chunk of items, a lane each: `bytes` is the lane's item length without the comma (0: no item); `put(w)` writes
    // it.  Returns whether any lane had an item.
    template <class Put>
    __device__ bool items(bool have, u32 bytes, bool any_before, Put put) {
        const unsigned m = __ballot_sync(LB_FULL, have);
        const bool comma = have && (any_before || (m & ((1u << lane) - 1u)));
        const u32 mine = have ? bytes + (comma ? 1u : 0u) : 0u;
        const u32 incl = (u32)warp_incl_scan((int)mine, lane);
        const u32 total = __shfl_sync(LB_FULL, incl, 31);
        if (out.dst && have) {
            Sink w;
            w.dst = out.dst; w.n = out.n + (incl - mine); w.flags = 0; w.wr = true;
            if (comma) w.put(',');
            put(w);
        }
        __syncwarp();
        out.n += total;
        return m != 0;
    }
    __device__ static void put_triple(Sink& w, u32 a, u32 b, u32 c) {
        w.put('['); Emitter::put_u32_to(w, a); w.put(','); Emitter::put_u32_to(w, b); w.put(','); Emitter::put_u32_to(w, c);
        w.put(']');
    }
    __device__ static u32 triple_len(u32 a, u32 b, u32 c) { return 4 + dec_digits(a) + dec_digits(b) + dec_digits(c); }

    // Text / List: the ids of the visible elements, merged into maximal runs
    __device__ void emit_runs(const DocContainer& dc) {
        out.put('[');
        const u32 n = dc.n_out;
        u32 prev_p = 0, open_c0 = 0;
        i32 prev_end = 0;
        bool any = false;
        for (u32 r0 = 0; r0 < n; r0 += 32) {
            const u32 r = r0 + (u32)lane;
            const bool valid = r < n;
            u32 p = 0;
            i32 c0 = 0, end = 0;
            if (valid) {
                const u32 row = t.out_row[dc.out0 + r];
                p = t.ch_peer[t.op_change[row]];
                c0 = t.op_counter[row] + (i32)t.out_off[dc.out0 + r];
                end = c0 + (i32)t.out_len[dc.out0 + r];
            }
            u32 pp = __shfl_up_sync(LB_FULL, p, 1);
            i32 pend = __shfl_up_sync(LB_FULL, end, 1);
            if (lane == 0) { pp = prev_p; pend = prev_end; }
            const bool start = valid && (r == 0 || pp != p || pend != c0);
            bool next_start = __shfl_down_sync(LB_FULL, start, 1);
            if (lane == 31 && r + 1 < n) {   // the run after the chunk
                const u32 row = t.out_row[dc.out0 + r + 1];
                next_start = t.ch_peer[t.op_change[row]] != p || t.op_counter[row] + (i32)t.out_off[dc.out0 + r + 1] != end;
            }
            const bool last = valid && (r + 1 == n || next_start);
            const unsigned sm_ = __ballot_sync(LB_FULL, start);
            const unsigned below = sm_ & ((2u << lane) - 1u);   // (2u << 31) - 1 wraps to every lane
            i32 g0 = __shfl_sync(LB_FULL, c0, below ? 31 - __clz((int)below) : 0);
            if (!below) g0 = (i32)open_c0;
            if (sm_) open_c0 = (u32)__shfl_sync(LB_FULL, c0, 31 - __clz((int)sm_));
            prev_p = __shfl_sync(LB_FULL, p, 31);
            prev_end = __shfl_sync(LB_FULL, end, 31);
            const u32 v = last ? vix(p) : 0;
            const u32 len = (u32)(end - g0);
            any |= items(last, last ? triple_len(v, (u32)g0, len) : 0, any, [&](Sink& w) { put_triple(w, v, (u32)g0, len); });
        }
        out.put(']');
    }

    __device__ bool map_has(u32 cidx) {
        bool has = false;
        for (u32 k = lane; k < di.K && !has; k += 32) has = t.map_best[di.mapslot0 + (u64)cidx * di.K + k] != 0;
        return __any_sync(LB_FULL, has);
    }
    // Map: every key whose winning op is inside the version, deletes included
    __device__ void emit_map(u32 cidx) {
        out.put('{');
        bool any = false;
        for (u32 k0 = 0; k0 < di.K; k0 += 32) {
            const u32 k = k0 + (u32)lane;
            bool have = false;
            u32 key = 0, v = 0, lam = 0, present = 0, bytes = 0;
            if (k < di.K) {
                key = kord[k];
                const u64 slot = di.mapslot0 + (u64)cidx * di.K + key;
                const unsigned long long best = t.map_best[slot];
                have = best != 0;
                if (have) {
                    const u32 row = t.map_row[slot];
                    present = t.op_kind[row] == OPK_MAP_SET;
                    lam = (u32)(best >> 32);
                    v = vix(t.ch_peer[t.op_change[row]]);
                    Sink cnt;
                    cnt.dst = nullptr; cnt.n = 0; cnt.flags = 0; cnt.wr = false;
                    cnt.put_escaped(t.bytes + t.dkey_off[di.key0 + key], t.dkey_len[di.key0 + key]);
                    bytes = 3 + (u32)cnt.n + triple_len(v, lam, present);
                }
            }
            any |= items(have, bytes, any, [&](Sink& w) {
                w.put('"');
                w.put_escaped(t.bytes + t.dkey_off[di.key0 + key], t.dkey_len[di.key0 + key]);
                w.put('"'); w.put(':');
                put_triple(w, v, lam, present);
            });
        }
        out.put('}');
    }

    // the tree op of node a's last effective move when the node belongs to tree container cidx, else 0xFFFFFFFF
    __device__ u32 node_move_row(u32 a, u32 cidx) const {
        if (t.tn_parent[di.tree0 + a] == TREE_UNEXIST) return 0xFFFFFFFFu;
        const u32 row = t.tr_rec[t.blocks[di.b0].tr0 + t.tn_move[di.tree0 + a]].w;
        return t.op_cidx[row] == cidx ? row : 0xFFFFFFFFu;
    }
    __device__ bool tree_has(u32 cidx) {
        if (!di.has_tree) return false;
        bool has = false;
        for (u32 a = lane; a < (u32)di.atom_total && !has; a += 32) has = node_move_row(a, cidx) != 0xFFFFFFFFu;
        return __any_sync(LB_FULL, has);
    }
    // Tree: every node the state holds, alive or deleted, by (peer, counter)
    __device__ void emit_tree(u32 cidx) {
        out.put('{');
        bool any = false;
        for (u32 r = 0; r < di.P; r++) {
            const u32 q = slot_of_rank(r);
            const DocPeer& dp = peer(q);
            const u32 qlen = id_len(q);
            for (u32 c0 = 0; c0 < (u32)dp.end_counter; c0 += 32) {
                const u32 ctr = c0 + (u32)lane;
                u32 row = 0xFFFFFFFFu;
                if (ctr < (u32)dp.end_counter) row = node_move_row(dp.atom_base + ctr, cidx);
                const bool have = row != 0xFFFFFFFFu;
                u32 v = 0, mc = 0, alive = 0, bytes = 0;
                if (have) {
                    v = vix(t.ch_peer[t.op_change[row]]);
                    mc = (u32)t.op_counter[row];
                    alive = t.tn_root[di.tree0 + dp.atom_base + ctr] != TREE_UNEXIST;
                    bytes = 4 + dec_digits(ctr) + qlen + triple_len(v, mc, alive);
                }
                any |= items(have, bytes, any, [&](Sink& w) {
                    w.put('"'); Emitter::put_u32_to(w, ctr); w.put('@'); put_id(w, q); w.put('"'); w.put(':');
                    put_triple(w, v, mc, alive);
                });
            }
        }
        out.put('}');
    }

    __device__ void run(bool sort) {
        load_peers();
        if (sort) sort_tables();
        __syncwarp();
        out.puts_("{\"peers\":[");
        bool first = true;
        for (u32 r = 0; r < di.P; r++) {
            const u32 q = slot_of_rank(r);
            if (peer(q).end_counter <= 0) continue;
            if (!first) out.put(',');
            first = false;
            out.put('"'); put_id(out, q); out.put('"');
        }
        out.puts_("],\"containers\":{");
        first = true;
        for (u32 i = 0; i < di.C; i++) {
            const u32 c = cord[i];
            const DocContainer& dc = t.dcont[di.cid0 + c];
            bool has;
            switch (dc.type) {
                case CT_TEXT: case CT_LIST: has = dc.n_out > 0; break;
                case CT_MAP: has = map_has(c); break;
                case CT_TREE: has = tree_has(c); break;
                default: has = false;   // MovableList / Counter: the document is unsupported
            }
            if (!has) continue;
            if (!first) out.put(',');
            first = false;
            out.put('"');
            put_cid_to(out, t, di, c, [&](u32 q) { put_id(out, q); });
            out.put('"'); out.put(':');
            if (dc.type == CT_MAP) emit_map(c);
            else if (dc.type == CT_TREE) emit_tree(c);
            else emit_runs(dc);
        }
        out.puts_("}}");
    }
};

// pass = 0: order the containers and keys, count bytes into len[d] ; pass = 1: write at off[d]
__global__ void __launch_bounds__(128) k_attr(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t,
                                             u32* __restrict__ cord, u32* __restrict__ kord, u32* __restrict__ len,
                                             const u64* __restrict__ off, u8* __restrict__ out, int pass) {
    __shared__ AttrSmem sm[4];   // 128 threads: one entry per warp
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // one warp per document
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK || di.has_unsupported) {   // the host answers "" for these (lb_doc_json's rule)
        if (!pass && lane == 0) len[d] = 0;
        return;
    }
    Sink s;
    s.dst = pass ? out + off[d] : nullptr;
    s.n = 0;
    s.flags = 0;
    s.wr = lane == 0;
    AttrWriter w(t, di, s, lane, &sm[(threadIdx.x >> 5) & 3], cord, kord);
    w.run(pass == 0);
    __syncwarp();
    if (!pass && lane == 0) len[d] = (u32)s.n;
}
