// loro_b200 -- cursors: where an element of a Text or List container lies now (LoroDoc::get_cursor_pos,
// crates/loro-internal/src/loro.rs:1560-1737), for any number of cursors of any documents in one call.
//
// Import time (LB_FLAG_CURSORS only), right after phase 5 and before its tracker pools are freed, k_cursor_tables runs
// a warp per document and keeps two tables per Text / List container, both based at the container's DocContainer::out0
// (out_cap bounds every span of the final rope, k_classify.cuh):
//   ord  every span of the final rope in document order, deleted spans included, the placeholder span not:
//        (peer index | CUR_VIS when visible, counter, length, visible atoms before the span) -- the order the
//        reference's tracker walks in get_target_id_latest_index_at_new_version (tracker.rs:588-619);
//   idx  the same spans by id: (doc-local atom index of the span's first id, its ord entry), ascending.  The atom index
//        of (peer, counter) is DocPeer::atom_base + counter, and the peers' atom ranges do not overlap, so ascending atom
//        index is ascending (peer, counter).  The order comes from a counting sort over the document's atom array: the
//        walk marks each span's first atom with its entry, then the warp reads the atoms in order and appends each mark
//        to its container's idx.
// Query time, k_cursor_query runs a warp per cursor: a ballot over the document's containers, a 32-way search of idx for
// the span holding the target id, and for a deleted target a 32-way search of ord for the visible element at its
// position (the update cursor).
#pragma once
#include "k_seq.cuh"

#define CUR_NONE 0xFFFFFFFFu
#define CUR_VIS 0x80000000u

struct CursorTables {
    uint4* ord;   // per container from out0: (peer | CUR_VIS, counter, len, visible atoms before)
    uint2* idx;   // per container from out0: (doc-local atom of the span's first id, entry of ord), ascending
    u32* n;       // per container: entries of ord and idx
};

// One cursor as the device reads it: lb_cursor with the root name moved into the call's name buffer.
struct CurReq {
    u64 doc;
    u64 cpeer;          // normal container: creator peer
    u64 tpeer;          // target id
    u64 name_off;       // root container: name bytes in the name buffer
    u32 name_len;
    i32 ccounter;       // normal container: creator counter
    i32 tctr;
    u8 is_root, type, has_id;
    int8_t side;
};

__global__ void __launch_bounds__(128)
k_cursor_tables(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ SeqPools pools,
                const __grid_constant__ BatchTables t, const __grid_constant__ CursorTables ct, u32* __restrict__ mark,
                u32* __restrict__ ent_cont, u32* __restrict__ fill) {
    const u32 d = (u32)(((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = (int)(threadIdx.x & 31);
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK || di.n_applied == 0 || di.C == 0) return;
    const DocPeer* dpeer = t.dpeer + di.peer0;
    const u64 doc_out0 = t.dcont[di.cid0].out0;   // the document's containers own consecutive out ranges
    const unsigned lt = (1u << lane) - 1;
    // ---- the final rope of every container, in document order; mark[first atom of a span] = doc-local entry
    for (u32 ci = 0; ci < di.C; ci++) {
        const DocContainer& dc = t.dcont[di.cid0 + ci];
        if (!dc.leaf_cap || dc.n_leaves == 0) continue;
        const u64 out0 = dc.out0;
        const u32 cap = dc.out_cap;
        u32 n = 0, before = 0;
        for (u32 leaf = dc.first_leaf; leaf != LEAF_NONE;) {
            uint4 L = pools.leaf[(dc.leaf0 + leaf) * 32 + lane];
            const u32 pe = L.x & 0xFFFFu;
            const bool real = pe != PEER_NONE && pe != PEER_UNKNOWN;
            const bool live = real && (L.x >> 16) == 0;
            const unsigned m = __ballot_sync(LB_FULL, real);
            const i32 v = live ? (i32)L.z : 0;
            const i32 incl = warp_incl_scan(v, lane);
            const u32 o = n + __popc(m & lt);
            if (real && o < cap) {
                ct.ord[out0 + o] = mk4(pe | (live ? CUR_VIS : 0u), L.y, L.z, before + (u32)(incl - v));
                mark[di.atom0 + dpeer[pe].atom_base + L.y] = (u32)(out0 - doc_out0) + o;
                ent_cont[out0 + o] = ci;
            }
            before += (u32)__shfl_sync(LB_FULL, incl, 31);
            n += __popc(m);
            leaf = __shfl_sync(LB_FULL, L.w, 1);
        }
        if (lane == 0) ct.n[di.cid0 + ci] = n < cap ? n : cap;
    }
    __syncwarp();
    // ---- counting sort: the marks in atom order, appended to their container's idx; one round per distinct container
    // among the 32 atoms at hand (almost always one)
    for (u64 a0 = 0; a0 < di.atom_total; a0 += 32) {
        const u64 a = a0 + (u64)lane;
        const u32 e = a < di.atom_total ? mark[di.atom0 + a] : CUR_NONE;
        const u32 c = e != CUR_NONE ? ent_cont[doc_out0 + e] : CUR_NONE;
        unsigned pend = __ballot_sync(LB_FULL, e != CUR_NONE);
        while (pend) {
            const u32 c0 = __shfl_sync(LB_FULL, c, __ffs(pend) - 1);
            const unsigned grp = __ballot_sync(LB_FULL, e != CUR_NONE && c == c0);
            const u64 out0 = t.dcont[di.cid0 + c0].out0;
            const u32 f = fill[di.cid0 + c0];
            if (grp & (1u << lane)) ct.idx[out0 + f + __popc(grp & lt)] = mk2((u32)a, (u32)(doc_out0 + e - out0));
            __syncwarp();
            if (lane == 0) fill[di.cid0 + c0] = f + __popc(grp);
            __syncwarp();
            pend &= ~grp;
        }
    }
}

// Number of entries k in [0, n) with key(k) <= x, for keys ascending in k: a 32-way search, every lane probes one point.
template <class Key>
__device__ __forceinline__ u32 cur_count_le(u32 n, u32 x, int lane, Key key) {
    u32 lo = 0, hi = n;   // the count lies in [lo, hi]
    while (lo < hi) {
        const u32 step = (hi - lo + 31) / 32;
        const u64 p = (u64)lo + (u64)(lane + 1) * step - 1;
        const bool le = p < hi && key((u32)p) <= x;
        const u32 k = (u32)__popc(__ballot_sync(LB_FULL, le));
        const u64 top = (u64)lo + (u64)(k + 1) * step - 1;
        lo += k * step;
        hi = top < hi ? (u32)top : hi;
    }
    return lo;
}

__device__ __forceinline__ bool cur_bytes_eq(const u8* a, const u8* b, u32 n) {
    for (u32 i = 0; i < n; i++)
        if (a[i] != b[i]) return false;
    return true;
}

// One warp per cursor.  The order of the checks is the reference's (loro.rs:1565-1737): the document, the container
// type the reference answers for, has_container, the visible element (state.rs:1403-1433), then the deleted one.
__global__ void __launch_bounds__(128)
k_cursor_query(const DocInfo* __restrict__ docs, const __grid_constant__ BatchTables t, const __grid_constant__ CursorTables ct,
               const CurReq* __restrict__ reqs, const u8* __restrict__ names, u64 n_reqs, lb_cursor_result* __restrict__ out) {
    const u64 r = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = (int)(threadIdx.x & 31);
    if (r >= n_reqs) return;
    const CurReq q = reqs[r];
    lb_cursor_result res;
    memset(&res, 0, sizeof(res));
    res.status = LB_OK;
    res.side = q.side;
    const DocInfo& di = docs[q.doc];
    const bool text_or_list = q.type == CT_TEXT || q.type == CT_LIST;
    if (di.code == DOC_ERR_UNSUPPORTED || (di.code == DOC_OK && di.has_unsupported)) res.status = LB_ERR_UNSUPPORTED;
    else if (di.code != DOC_OK || !text_or_list || q.side < -1 || q.side > 1) res.status = LB_ERR_INVALID_ARG;
    else {
        u32 ci = CUR_NONE;
        for (u32 c0 = 0; c0 < di.C && ci == CUR_NONE; c0 += 32) {
            const u32 c = c0 + (u32)lane;
            bool hit = false;
            if (c < di.C) {
                const DocContainer& dc = t.dcont[di.cid0 + c];
                if (dc.is_root == q.is_root && dc.type == q.type) {
                    if (q.is_root) hit = dc.name_len == q.name_len && cur_bytes_eq(t.bytes + dc.name_off, names + q.name_off, q.name_len);
                    else hit = dc.peer == q.cpeer && dc.counter == q.ccounter;
                }
            }
            const unsigned m = __ballot_sync(LB_FULL, hit);
            if (m) ci = c0 + (u32)(__ffs(m) - 1);
        }
        // a root container always exists (loro.rs:889-896); one that no op touches is empty
        u32 len = 0, n = 0;
        u64 out0 = 0;
        if (ci != CUR_NONE) {
            const DocContainer& dc = t.dcont[di.cid0 + ci];
            len = dc.seq_len;
            n = ct.n[di.cid0 + ci];
            out0 = dc.out0;
        }
        const DocPeer* dpeer = t.dpeer + di.peer0;
        if (ci == CUR_NONE && !q.is_root) res.status = LB_CURSOR_ID_NOT_FOUND;
        else if (!q.has_id) res.pos = q.side == -1 ? 0 : len;
        else {
            u32 pi = CUR_NONE;
            for (u32 p0 = 0; p0 < di.P && pi == CUR_NONE; p0 += 32) {
                const u32 p = p0 + (u32)lane;
                const unsigned m = __ballot_sync(LB_FULL, p < di.P && dpeer[p].id == q.tpeer);
                if (m) pi = p0 + (u32)(__ffs(m) - 1);
            }
            bool found = false;
            uint4 E = mk4(0, 0, 0, 0);
            u32 off = 0;
            if (pi != CUR_NONE && q.tctr >= 0 && q.tctr < dpeer[pi].end_counter) {
                const u32 a = dpeer[pi].atom_base + (u32)q.tctr;
                const uint2* idx = ct.idx + out0;
                const u32 k = cur_count_le(n, a, lane, [&](u32 j) { return idx[j].x; });
                if (k) {
                    const uint2 s = idx[k - 1];
                    E = ct.ord[out0 + s.y];
                    off = a - s.x;
                    found = off < E.z;
                }
            }
            if (!found) res.status = LB_CURSOR_ID_NOT_FOUND;
            else if (E.x & CUR_VIS) res.pos = E.w + off;
            else {
                // deleted: the visible elements before it, Side::Left, and get_cursor(pos, Left) on the current state
                // (handler.rs:2337-2390 Text, :2912-2952 List)
                const u32 pos = E.w;
                res.pos = pos;
                res.side = -1;
                res.has_update = 1;
                res.update_side = -1;
                if (len == 0) res.update_origin_pos = 0;
                else if (pos >= len) { res.update_side = 1; res.update_origin_pos = len; }
                else {
                    const uint4* ord = ct.ord + out0;
                    const u32 j = cur_count_le(n, pos, lane, [&](u32 k) {
                        const uint4 x = ord[k];
                        return x.w + ((x.x & CUR_VIS) ? x.z : 0u);
                    });
                    const uint4 V = ord[j];
                    res.update_has_id = 1;
                    res.update_peer = dpeer[V.x & 0xFFFFu].id;
                    res.update_counter = (i32)V.y + (i32)(pos - V.w);
                    res.update_origin_pos = pos;
                }
            }
        }
    }
    if (lane == 0) out[r] = res;
}
