// loro_b200 -- phase 5: eg-walker (Fugue) integration of List/Text containers, one warp per document at a time.
//
// Replaces (reference, relative to crates/loro-internal/src):
//   container/richtext/tracker.rs:84-232 (insert/delete), :330-526 (checkout: retreat / forward)
//   container/richtext/tracker/crdt_rope.rs:43-227 (Fugue origin reconstruction + sibling scan),
//     :236-315 (delete), :325-361 (status updates), :542-652 (active-length queries)
//   container/richtext/fugue_span.rs:192-386 (span status: future / delete_times ; slicing)
//   container/richtext/tracker/id_to_cursor.rs (id -> span lookup)  ->  dense atom -> leaf array
//   diff_calc.rs:175-236,585-620 (per-change checkout then apply)
//
// Data structure: per container a B+tree.
//   * leaves (HBM): 32 slots of one uint4 (peer | state << 16, counter, len, aux); lane i of the warp owns slot i,
//     so a whole leaf -- spans, parent link (aux of slot 0) and next-leaf link (aux of slot 1) -- arrives with ONE
//     128-bit load per lane, and "k-th visible atom" is a shuffle scan + ballot.  Unused slots hold a sentinel,
//     so no count has to be read before the slots;
//   * internal nodes: 32 (child, visible-length) pairs; the first NS nodes of the active container live in
//     SHARED memory (one private region per warp), the rest spill to HBM;
//   * per document, dense atom-indexed arrays (HBM): atom -> leaf and the Fugue origins of every span start
//     (one uint4).  Spans never merge or disappear, they only split, and a split never moves atoms, so only a
//     leaf split rewrites atom -> leaf entries.
// The kernel is bound by the latency of dependent HBM loads, so everything that can
// be looked up ahead is fetched lane-parallel: 32 change headers, 32 op records, the 32 target leaves of a
// version switch are each one round trip, and the warp then consumes them with shuffles.
// Deletes are applied by target id (for well-formed histories the reference's by-position deletion hits the
// same atoms).  Every function is warp-synchronous: all 32 lanes call it with identical arguments; a
// __syncwarp() separates reads by all lanes from a following write by one lane to the same location.
// Rare paths (splits, the sibling scan) are separate __noinline__ functions working on per-warp state in
// shared memory: the v2 kernel inlined them everywhere and stalled on instruction fetch (44k SASS lines).
#pragma once
#include "lb_tables.cuh"

#define NODE_NONE 0xFFFFFFFFu
#define LEAF_NONE 0xFFFFFFFFu
#define ST_FUTURE 0x8000u
#define SLOT_EMPTY ((u32)PEER_NONE | (1u << 16))   // no peer, never visible
#define LB_SEQ_NS 12          // internal nodes cached in shared memory per warp
#define LB_SEQ_WARPS 4        // warps (documents) per CTA

// op record written by k_op_classify: x = kind | reversed << 3 | container << 4, y = counter, z = atoms,
// w = insert position (SEQ_INS) or lowest target counter (SEQ_DEL); op_aux = target peer of a delete
#define REC_KIND(x) ((x) & 7u)
#define REC_REV(x) (((x) >> 3) & 1u)
#define REC_CIDX(x) ((x) >> 4)

struct SeqPools {
    uint4* leaf;         // [leaf][32]
    uint2* node;         // [node][32] (child, visible atoms below)   (global home of the nodes)
    u32* node_parent;    // (parent << 5) | index inside the parent, NODE_NONE for the root
    u32* atom_leaf;      // LEAF_NONE = not an inserted list/text atom (yet)
    uint4* a_org;        // origins, valid at span starts: x = ol_peer | or_peer << 16, y = ol_ctr, z = or_ctr
    i32* cvv;            // per container: tracker current_vv (P entries)
    u32* cont_epoch;     // per container: last walk index that checked out / applied an op
    u32* next_doc;       // the launch's work queue: index of the next document to hand to a warp (zero at launch)
};

struct SeqSmem {   // one per warp
    u32 child[LB_SEQ_NS][32];
    i32 vis[LB_SEQ_NS][32];
    u32 parent[LB_SEQ_NS];
    u32 abase[32];     // atom_base of the document's first 32 peers
    i32 cvv[32];       // tracker version of the active container, first 32 peers
    // The same for all 32 lanes and changed only per document or per container switch: kept here rather than in
    // registers, where every helper call would carry them and the kernel spilled them at its register budget.
    const DocPeer* dpeer;   // the document's peers
    u64 atom0;              // the document's first atom
    u64 leaf0, node0, cvv0; // pool bases of the active container
    u32 P;                  // the document's peers
    // active container
    u32 root, height, first_leaf, n_leaves, n_nodes, unk_leaf, leaf_cap, node_cap;
    u32 err;
};

// The warp's SeqSmem.  The __noinline__ helpers take it from here instead of as an argument: a shared-memory address
// computed from the thread index needs no register across a call.
__shared__ SeqSmem seq_smem[LB_SEQ_WARPS];
__device__ __forceinline__ SeqSmem* seq_sm() { return &seq_smem[threadIdx.x >> 5]; }
__device__ __forceinline__ int seq_lane() { return (int)(threadIdx.x & 31); }

__device__ __forceinline__ uint4 mk4(u32 x, u32 y, u32 z, u32 w) { uint4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
__device__ __forceinline__ uint2 mk2(u32 x, u32 y) { uint2 r; r.x = x; r.y = y; return r; }
__device__ __forceinline__ void seq_fail(SeqSmem* sm, u32 code) {
    if (seq_lane() == 0 && sm->err == 0) sm->err = code;
    __syncwarp();
}
__device__ __forceinline__ u64 atom_index(SeqSmem* sm, u32 peer, i32 ctr) {
    u32 base = peer < 32 ? sm->abase[peer] : sm->dpeer[peer].atom_base;
    return sm->atom0 + base + (u32)ctr;
}
__device__ __forceinline__ i32 cvv_get(const SeqPools& p, SeqSmem* sm, u32 q) { return q < 32 ? sm->cvv[q] : p.cvv[sm->cvv0 + q]; }
__device__ __forceinline__ void cvv_set(const SeqPools& p, SeqSmem* sm, u32 q, i32 v) { if (q < 32) sm->cvv[q] = v; else p.cvv[sm->cvv0 + q] = v; }

// ---- slots
__device__ __forceinline__ u32 s_peer(const uint4& s) { return s.x & 0xFFFFu; }
__device__ __forceinline__ u32 s_st(const uint4& s) { return s.x >> 16; }
__device__ __forceinline__ i32 s_vis(const uint4& s) { return (s.x >> 16) == 0 ? (i32)s.z : 0; }
__device__ __forceinline__ uint4 leaf_load(const SeqPools& p, SeqSmem* sm, u32 leaf) { return p.leaf[(sm->leaf0 + leaf) * 32 + seq_lane()]; }
// slots below `from` are unchanged by the caller: only the shifted tail goes back to HBM
__device__ __forceinline__ void leaf_store(const SeqPools& p, SeqSmem* sm, u32 leaf, const uint4& L, int from = 0) {
    if (seq_lane() >= from) p.leaf[(sm->leaf0 + leaf) * 32 + seq_lane()] = L;
    __syncwarp();
}
__device__ __forceinline__ int leaf_count(const uint4& L) { return __popc(__ballot_sync(LB_FULL, s_peer(L) != PEER_NONE)); }
// slot of the span containing atom (peer, ctr) inside a loaded leaf image, -1 when absent
__device__ __forceinline__ int slot_of(const uint4& L, u32 peer, i32 ctr) {
    unsigned m = __ballot_sync(LB_FULL, s_peer(L) == peer && ctr >= (i32)L.y && ctr < (i32)L.y + (i32)L.z);
    return __ffs(m) - 1;
}

// ---- nodes (shared-memory cache for ids < NS)
__device__ __forceinline__ uint2 nd_get(const SeqPools& p, SeqSmem* sm, u32 nd, int i) {
    return nd < LB_SEQ_NS ? mk2(sm->child[nd][i], (u32)sm->vis[nd][i]) : p.node[(sm->node0 + nd) * 32 + i];
}
__device__ __forceinline__ void nd_set(const SeqPools& p, SeqSmem* sm, u32 nd, int i, u32 child, i32 vis) {
    if (nd < LB_SEQ_NS) { sm->child[nd][i] = child; sm->vis[nd][i] = vis; }
    else p.node[(sm->node0 + nd) * 32 + i] = mk2(child, (u32)vis);
}
__device__ __forceinline__ u32 nd_parent(const SeqPools& p, SeqSmem* sm, u32 nd) {
    return nd < LB_SEQ_NS ? sm->parent[nd] : p.node_parent[sm->node0 + nd];
}
__device__ __forceinline__ void nd_set_parent(const SeqPools& p, SeqSmem* sm, u32 nd, u32 v) {
    if (nd < LB_SEQ_NS) sm->parent[nd] = v; else p.node_parent[sm->node0 + nd] = v;
}
__device__ __forceinline__ void nd_add_vis(const SeqPools& p, SeqSmem* sm, u32 nd, int i, i32 d) {
    if (nd < LB_SEQ_NS) sm->vis[nd][i] += d;
    else { uint2* q = &p.node[(sm->node0 + nd) * 32 + i]; q->y = (u32)((i32)q->y + d); }
}
__device__ __forceinline__ void set_child_link(const SeqPools& p, SeqSmem* sm, bool kids_are_leaves, u32 child, u32 link) {
    if (kids_are_leaves) p.leaf[(sm->leaf0 + child) * 32].w = link; else nd_set_parent(p, sm, child, link);
}
// add `delta` visible atoms on the path (parent link of a leaf) -> root
__device__ __forceinline__ void add_vis(const SeqPools& p, SeqSmem* sm, u32 link, i32 delta) {
    if (delta != 0 && seq_lane() == 0) {
        while (link != NODE_NONE) {
            u32 nd = link >> 5;
            nd_add_vis(p, sm, nd, (int)(link & 31), delta);
            link = nd_parent(p, sm, nd);
        }
    }
    __syncwarp();
}

// ---- insert (child, vis) into node `nd` right after index `after`; room must exist
__device__ __forceinline__ void node_insert_no_split(const SeqPools& p, SeqSmem* sm, u32 nd, int after, u32 child, i32 vis,
                                                     bool kids_are_leaves) {
    int lane = seq_lane();
    uint2 e = nd_get(p, sm, nd, lane);
    int n = __popc(__ballot_sync(LB_FULL, e.x != NODE_NONE));
    u32 c_up = __shfl_up_sync(LB_FULL, e.x, 1);
    u32 v_up = __shfl_up_sync(LB_FULL, e.y, 1);
    int at = after + 1;
    if (lane == at) { e.x = child; e.y = (u32)vis; }
    else if (lane > at) { e.x = c_up; e.y = v_up; }
    __syncwarp();
    if (lane <= n) nd_set(p, sm, nd, lane, e.x, (i32)e.y);
    if (lane >= at && lane <= n) set_child_link(p, sm, kids_are_leaves, e.x, (nd << 5) | (u32)lane);
    __syncwarp();
}
__device__ __forceinline__ i32 node_total(const SeqPools& p, SeqSmem* sm, u32 nd) {
    return warp_sum((i32)nd_get(p, sm, nd, seq_lane()).y);
}
// ---- insert with splits propagating upward
__device__ __noinline__ void node_insert(const SeqPools& p, u32 nd, int after, u32 child, i32 vis, bool kids_are_leaves) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    while (true) {
        uint2 e = nd_get(p, sm, nd, lane);
        int n = __popc(__ballot_sync(LB_FULL, e.x != NODE_NONE));
        if (n < 32) { node_insert_no_split(p, sm, nd, after, child, vis, kids_are_leaves); return; }
        if (sm->n_nodes >= sm->node_cap) { seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY)); return; }
        __syncwarp();
        u32 nn = sm->n_nodes;
        __syncwarp();
        if (lane == 0) sm->n_nodes = nn + 1;
        // upper half moves to the new node
        u32 uc = __shfl_down_sync(LB_FULL, e.x, 16);
        u32 uv = __shfl_down_sync(LB_FULL, e.y, 16);
        if (lane < 16) {
            nd_set(p, sm, nn, lane, uc, (i32)uv);
            set_child_link(p, sm, kids_are_leaves, uc, (nn << 5) | (u32)lane);
        } else {
            nd_set(p, sm, nn, lane, NODE_NONE, 0);
            nd_set(p, sm, nd, lane, NODE_NONE, 0);
        }
        __syncwarp();
        if (after >= 16) node_insert_no_split(p, sm, nn, after - 16, child, vis, kids_are_leaves);
        else node_insert_no_split(p, sm, nd, after, child, vis, kids_are_leaves);
        i32 tot_old = node_total(p, sm, nd), tot_new = node_total(p, sm, nn);
        u32 plink = nd_parent(p, sm, nd);
        __syncwarp();   // every lane has read the parent link before it is rewritten
        if (plink == NODE_NONE) {
            if (sm->n_nodes >= sm->node_cap) { seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY)); return; }
            __syncwarp();
            u32 nr = sm->n_nodes;
            u32 h = sm->height;
            __syncwarp();
            nd_set(p, sm, nr, lane, lane == 0 ? nd : (lane == 1 ? nn : NODE_NONE), lane == 0 ? tot_old : (lane == 1 ? tot_new : 0));
            if (lane == 0) {
                nd_set_parent(p, sm, nr, NODE_NONE);
                nd_set_parent(p, sm, nd, (nr << 5) | 0u);
                nd_set_parent(p, sm, nn, (nr << 5) | 1u);
                sm->n_nodes = nr + 1;
                sm->root = nr;
                sm->height = h + 1;
            }
            __syncwarp();
            return;
        }
        u32 parent = plink >> 5;
        int idx = (int)(plink & 31);
        if (lane == 0) nd_set(p, sm, parent, idx, nd, tot_old);
        __syncwarp();
        child = nn;
        vis = tot_new;
        after = idx;
        nd = parent;
        kids_are_leaves = false;
    }
}

// ---- split a full leaf: upper 16 slots move to a new leaf (their atom -> leaf entries follow)
__device__ __noinline__ void leaf_split(const SeqPools& p, u32 leaf) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    if (sm->n_leaves >= sm->leaf_cap) { seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY)); return; }
    __syncwarp();
    u32 nl = sm->n_leaves;
    __syncwarp();
    if (lane == 0) sm->n_leaves = nl + 1;
    uint4 L = leaf_load(p, sm, leaf);
    u32 link = __shfl_sync(LB_FULL, L.w, 0);
    u32 next = __shfl_sync(LB_FULL, L.w, 1);
    uint4 U;
    U.x = __shfl_down_sync(LB_FULL, L.x, 16);
    U.y = __shfl_down_sync(LB_FULL, L.y, 16);
    U.z = __shfl_down_sync(LB_FULL, L.z, 16);
    U.w = lane == 1 ? next : 0;   // parent link (slot 0) is set by node_insert below
    if (lane >= 16) { U.x = SLOT_EMPTY; U.y = 0; U.z = 0; }
    __syncwarp();
    p.leaf[(sm->leaf0 + nl) * 32 + lane] = U;
    uint4 O = L;
    if (lane >= 16) { O.x = SLOT_EMPTY; O.y = 0; O.z = 0; }
    if (lane == 1) O.w = nl;
    p.leaf[(sm->leaf0 + leaf) * 32 + lane] = O;
    // atoms of the moved spans get their new home
    u32 pe = s_peer(L);
    bool moved_real = lane >= 16 && pe != PEER_NONE && pe != PEER_UNKNOWN;
    if (moved_real) p.atom_leaf[atom_index(sm, pe, (i32)L.y)] = nl;
    unsigned longm = __ballot_sync(LB_FULL, moved_real && (i32)L.z > 1);
    while (longm) {
        int s = __ffs(longm) - 1;
        longm &= longm - 1;
        u32 sp = __shfl_sync(LB_FULL, pe, s);
        i32 sc = (i32)__shfl_sync(LB_FULL, L.y, s);
        i32 sl = (i32)__shfl_sync(LB_FULL, L.z, s);
        u64 a0 = atom_index(sm, sp, sc);
        for (i32 i = 1 + lane; i < sl; i += 32) p.atom_leaf[a0 + i] = nl;
    }
    unsigned unk = __ballot_sync(LB_FULL, lane >= 16 && pe == PEER_UNKNOWN);
    if (unk && lane == 0) sm->unk_leaf = nl;
    i32 moved = warp_sum(lane >= 16 ? s_vis(L) : 0);
    u32 parent = link >> 5;
    int idx = (int)(link & 31);
    if (lane == 0) nd_add_vis(p, sm, parent, idx, -moved);
    __syncwarp();
    node_insert(p, parent, idx, nl, moved, true);
}

// ---- split the span containing atom (peer, ctr) right before that atom (FugueSpan::_slice,
// fugue_span.rs:257-279); visible totals unchanged.  No-op when (peer, ctr) already starts a span.
__device__ __noinline__ void split_before(const SeqPools& p, u32 peer, i32 ctr) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    for (int attempt = 0; attempt < 2; attempt++) {
        u32 leaf = p.atom_leaf[atom_index(sm, peer, ctr)];
        if (leaf == LEAF_NONE) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }
        uint4 L = leaf_load(p, sm, leaf);
        int slot = slot_of(L, peer, ctr);
        if (slot < 0) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }
        i32 s_ctr = (i32)__shfl_sync(LB_FULL, L.y, slot);
        if (s_ctr == ctr) return;
        if (leaf_count(L) >= 32) {   // make room first; the span (still whole) may move to the new leaf
            if (attempt) { seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY)); return; }
            leaf_split(p, leaf);
            if (sm->err) return;
            continue;
        }
        i32 s_len = (i32)__shfl_sync(LB_FULL, L.z, slot);
        u32 s_x = __shfl_sync(LB_FULL, L.x, slot);
        i32 k = ctr - s_ctr;
        u32 ux = __shfl_up_sync(LB_FULL, L.x, 1);
        u32 uy = __shfl_up_sync(LB_FULL, L.y, 1);
        u32 uz = __shfl_up_sync(LB_FULL, L.z, 1);
        if (lane == slot) L.z = (u32)k;                       // left part keeps its slot
        else if (lane == slot + 1) { L.x = s_x; L.y = (u32)ctr; L.z = (u32)(s_len - k); }
        else if (lane > slot + 1) { L.x = ux; L.y = uy; L.z = uz; }
        leaf_store(p, sm, leaf, L, slot);
        // origins of the new span start: left origin is its predecessor, right origin is inherited
        uint4 og = p.a_org[atom_index(sm, peer, s_ctr)];
        if (lane == 0) p.a_org[atom_index(sm, peer, ctr)] = mk4(peer | (og.x & 0xFFFF0000u), (u32)(ctr - 1), og.z, 0);
        __syncwarp();
        return;
    }
}

// ---- apply a status change to the inserted atoms [t0,t1) of `peer`: set_future 1/0/-1 (set, clear, keep),
// del_diff added to the delete counter.  `hint` is a (possibly stale) atom -> leaf lookup of (peer, t0).
__device__ __noinline__ void range_apply(const SeqPools& p, u32 peer, i32 t0, i32 t1, int set_future, int del_diff, u32 hint) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    i32 cur = t0;
    u32 leaf = hint;
    int guard = 0;
    while (cur < t1) {
        if (leaf == LEAF_NONE) {
            leaf = p.atom_leaf[atom_index(sm, peer, cur)];
            if (leaf == LEAF_NONE) { cur++; continue; }   // never integrated here (foreign container)
        }
        uint4 L = leaf_load(p, sm, leaf);
        int slot = slot_of(L, peer, cur);
        if (slot < 0) {            // stale hint (a leaf split moved the span): look the atom up again
            if (++guard > 2) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }
            leaf = LEAF_NONE;
            continue;
        }
        i32 s_ctr = (i32)__shfl_sync(LB_FULL, L.y, slot);
        i32 s_len = (i32)__shfl_sync(LB_FULL, L.z, slot);
        if (s_ctr != cur || cur + s_len > t1) {
            // boundaries do not line up with the span: cut it, then look again
            if (s_ctr != cur) split_before(p, peer, cur);
            if (!sm->err && s_ctr + s_len > t1) split_before(p, peer, t1);
            if (sm->err) return;
            leaf = LEAF_NONE;
            guard = 0;
            continue;
        }
        // every span of the chain cur, cur+len, ... that lives in this leaf and ends inside the range
        bool mine = false;
        while (true) {
            unsigned m = __ballot_sync(LB_FULL, s_peer(L) == peer && (i32)L.y == cur && cur + (i32)L.z <= t1);
            if (!m) break;
            int s = __ffs(m) - 1;
            if (lane == s) mine = true;
            cur += (i32)__shfl_sync(LB_FULL, L.z, s);
        }
        i32 before = mine ? s_vis(L) : 0;
        if (mine) {
            u32 st = s_st(L);
            if (set_future == 1) st |= ST_FUTURE;
            if (set_future == 0) st &= ~ST_FUTURE;
            st = (st & ST_FUTURE) | (((st & 0x7FFFu) + (u32)del_diff) & 0x7FFFu);
            L.x = (L.x & 0xFFFFu) | (st << 16);
            p.leaf[(sm->leaf0 + leaf) * 32 + lane].x = L.x;
        }
        i32 delta = warp_sum((mine ? s_vis(L) : 0) - before);
        add_vis(p, sm, __shfl_sync(LB_FULL, L.w, 0), delta);
        leaf = LEAF_NONE;
        guard = 0;
    }
}

// ---- lane-local status change: every lane applies its OWN range [t0,t1) of `peer` with atomics (state word of
// the slot, visible lengths on the path to the root), so 32 ranges proceed at once and their dependent loads
// overlap.  Handles the spans that line up with the range; returns the first counter that needs the
// warp-cooperative path (a span must be cut, or the atom is unknown here), t1 when done.  No structure
// changes happen while lanes run this, so the hints taken at the start of the batch stay valid.
__device__ __forceinline__ i32 toggle_lane(const SeqPools& p, SeqSmem* sm, u32 peer, i32 t0, i32 t1, int set_future, int del_diff,
                                           u32 hint) {
    i32 cur = t0;
    u32 leaf = hint;
    while (cur < t1) {
        if (leaf == LEAF_NONE) {
            leaf = p.atom_leaf[atom_index(sm, peer, cur)];
            if (leaf == LEAF_NONE) return cur;
        }
        uint4* base = p.leaf + (sm->leaf0 + leaf) * 32;
        int found = -1;
        uint4 sl = mk4(0, 0, 0, 0);
        u32 link = NODE_NONE;
#pragma unroll 1
        for (int s0 = 0; s0 < 32 && found < 0; s0 += 4) {
            uint4 v0 = base[s0], v1 = base[s0 + 1], v2 = base[s0 + 2], v3 = base[s0 + 3];
            if (s0 == 0) link = v0.w;
            if ((v0.x & 0xFFFFu) == peer && cur >= (i32)v0.y && cur < (i32)(v0.y + v0.z)) { found = s0; sl = v0; }
            else if ((v1.x & 0xFFFFu) == peer && cur >= (i32)v1.y && cur < (i32)(v1.y + v1.z)) { found = s0 + 1; sl = v1; }
            else if ((v2.x & 0xFFFFu) == peer && cur >= (i32)v2.y && cur < (i32)(v2.y + v2.z)) { found = s0 + 2; sl = v2; }
            else if ((v3.x & 0xFFFFu) == peer && cur >= (i32)v3.y && cur < (i32)(v3.y + v3.z)) { found = s0 + 3; sl = v3; }
            else if ((v3.x & 0xFFFFu) == PEER_NONE) break;   // slots are compact: nothing further
        }
        if (found < 0) return cur;
        i32 len = (i32)sl.z;
        if ((i32)sl.y != cur || cur + len > t1) return cur;
        u32* word = &base[found].x;
        u32 old, nw;
        if (set_future == 1) { old = atomicOr(word, (u32)ST_FUTURE << 16); nw = old | ((u32)ST_FUTURE << 16); }
        else if (set_future == 0) { old = atomicAnd(word, ~((u32)ST_FUTURE << 16)); nw = old & ~((u32)ST_FUTURE << 16); }
        else { u32 d = (u32)del_diff << 16; old = atomicAdd(word, d); nw = old + d; }
        i32 delta = ((nw >> 16) == 0 ? len : 0) - ((old >> 16) == 0 ? len : 0);
        if (delta != 0) {
            while (link != NODE_NONE) {
                u32 nd = link >> 5;
                int idx = (int)(link & 31);
                if (nd < LB_SEQ_NS) atomicAdd(&sm->vis[nd][idx], delta);
                else atomicAdd((i32*)&p.node[(sm->node0 + nd) * 32 + idx].y, delta);
                link = nd_parent(p, sm, nd);
            }
        }
        cur += len;
        leaf = LEAF_NONE;
    }
    return cur;
}

// ---- retreat (dir=-1) / forward (dir=+1) the ops of peer `q` with counters [a,b) that touch container `cidx`.
// The peer's changes covering [a,b) are enumerated 32 at a time, their op rows flattened over the lanes, so the
// op records and the atom -> leaf lookups of 32 rows cost one round trip each.
__device__ __noinline__ void toggle_ops(const SeqPools& p, const BatchTables& t, u64 ch0, u32 cidx, u32 q, i32 a, i32 b, int dir) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    u32 row_a = t.atom_row[atom_index(sm, q, a)], row_b = t.atom_row[atom_index(sm, q, b - 1)];
    u32 pos_a = t.ch_pos[t.op_change[row_a]], pos_b = t.ch_pos[t.op_change[row_b]];
    for (u32 pb = pos_a; pb <= pos_b && !sm->err; pb += 32) {
        u32 pos = pb + (u32)lane;
        bool cv = pos <= pos_b;
        u32 ch = cv ? t.ch_aorder[ch0 + pos] : 0;
        u32 r0 = cv ? (u32)t.ch_op0[ch] : 0;
        i32 nr = cv ? (i32)t.ch_nops[ch] : 0;
        i32 incl = warp_incl_scan(nr, lane);
        i32 total = __shfl_sync(LB_FULL, incl, 31);
        i32 excl = incl - nr;
        for (i32 g0 = 0; g0 < total && !sm->err; g0 += 32) {
            i32 g = g0 + lane;
            bool gv = g < total;
            int j = 0;   // change of flat row g: number of lanes whose inclusive count is <= g
#pragma unroll
            for (int s = 16; s; s >>= 1) {
                i32 v = __shfl_sync(LB_FULL, incl, (j + s - 1) & 31);
                if (v <= g) j += s;
            }
            j &= 31;
            u32 row = __shfl_sync(LB_FULL, r0, j);
            i32 row_excl = __shfl_sync(LB_FULL, excl, j);
            row += (u32)(g - row_excl);
            uint4 rec = mk4(0, 0, 0, 0);
            u32 aux = 0;
            if (gv) { rec = t.op_rec[row]; aux = t.op_aux[row]; }
            u32 kind = REC_KIND(rec.x);
            i32 rc = (i32)rec.y, rn = (i32)rec.z;
            i32 c0 = rc > a ? rc : a, c1 = rc + rn < b ? rc + rn : b;
            bool act = gv && (kind == OPK_SEQ_INS || kind == OPK_SEQ_DEL) && REC_CIDX(rec.x) == cidx && c0 < c1;
            u32 tp = q;
            i32 t0 = c0, t1 = c1;
            int mode = dir < 0 ? 1 : 0;          // inserts: set / clear the future flag ; deletes: keep it, count
            int dd = 0;
            if (kind == OPK_SEQ_DEL) {
                tp = aux;
                i32 tc = (i32)rec.w;
                if (!REC_REV(rec.x)) { t0 = tc + (c0 - rc); t1 = tc + (c1 - rc); }
                else { t0 = tc + (rn - (c1 - rc)); t1 = tc + (rn - (c0 - rc)); }
                mode = -1;
                dd = dir;
            }
            u32 hint = act ? p.atom_leaf[atom_index(sm, tp, t0)] : LEAF_NONE;
            // lane-parallel: each lane flips the spans of its own row; what needs a cut comes back for the warp
            i32 done = t1;
            if (act) done = toggle_lane(p, sm, tp, t0, t1, mode, dd, hint);
            __syncwarp();
            unsigned m = __ballot_sync(LB_FULL, act && done < t1);
            while (m && !sm->err) {
                int s = __ffs(m) - 1;
                m &= m - 1;
                range_apply(p, __shfl_sync(LB_FULL, tp, s), __shfl_sync(LB_FULL, done, s), __shfl_sync(LB_FULL, t1, s),
                            __shfl_sync(LB_FULL, mode, s), __shfl_sync(LB_FULL, dd, s), LEAF_NONE);
            }
        }
    }
}

// ---- move the tracker of the active container to version vv (+ the author's own counter)
__device__ __forceinline__ void checkout(const SeqPools& p, const BatchTables& t, SeqSmem* sm, u64 ch0, u32 cidx, const i32* vv,
                                         u32 own_peer, i32 own_ctr) {
    int lane = seq_lane();
    for (u32 q0 = 0; q0 < sm->P && !sm->err; q0 += 32) {
        u32 q = q0 + (u32)lane;
        i32 tgt = 0, cur = 0;
        if (q < sm->P) {
            tgt = vv ? vv[q] : 0;
            if (q == own_peer && own_ctr > tgt) tgt = own_ctr;
            cur = cvv_get(p, sm, q);
        }
        unsigned m = __ballot_sync(LB_FULL, cur != tgt);
        while (m && !sm->err) {
            int s = __ffs(m) - 1;
            m &= m - 1;
            i32 cu = __shfl_sync(LB_FULL, cur, s), tg = __shfl_sync(LB_FULL, tgt, s);
            if (cu > tg) toggle_ops(p, t, ch0, cidx, q0 + (u32)s, tg, cu, -1);
            else toggle_ops(p, t, ch0, cidx, q0 + (u32)s, cu, tg, +1);
        }
        __syncwarp();
        if (q < sm->P && cur != tgt) cvv_set(p, sm, q, tgt);
        __syncwarp();
    }
}

// ---- position key of slot (leaf, slot) for cmp_pos (crdt_rope.rs:433-446)
__device__ __forceinline__ u64 order_key(const SeqPools& p, SeqSmem* sm, u32 leaf, int slot) {
    u64 key = (u64)slot;
    int shift = 6;
    u32 link = p.leaf[(sm->leaf0 + leaf) * 32].w;
    while (link != NODE_NONE) {
        key |= (u64)(link & 31) << shift;
        shift += 6;
        link = nd_parent(p, sm, link >> 5);
    }
    return key;
}
__device__ __forceinline__ u64 order_key_of_atom(const SeqPools& p, SeqSmem* sm, u32 peer, i32 ctr) {
    u32 leaf;
    uint4 L;
    int slot;
    if (peer == PEER_UNKNOWN) {
        leaf = sm->unk_leaf;
        L = leaf_load(p, sm, leaf);
        slot = __ffs(__ballot_sync(LB_FULL, s_peer(L) == PEER_UNKNOWN)) - 1;
    } else {
        leaf = p.atom_leaf[atom_index(sm, peer, ctr)];
        L = leaf_load(p, sm, leaf);
        slot = slot_of(L, peer, ctr);
    }
    return order_key(p, sm, leaf, slot);
}
// origin_left of atom (peer, ctr): stored for span starts, implied inside a span
__device__ __forceinline__ void atom_origin_left(const SeqPools& p, SeqSmem* sm, u32 peer, i32 ctr, u32* op, i32* oc) {
    if (peer == PEER_UNKNOWN) { *op = PEER_NONE; *oc = -1; return; }
    u64 ai = atom_index(sm, peer, ctr);
    u32 leaf = p.atom_leaf[ai];
    uint4 L = leaf_load(p, sm, leaf);
    int slot = slot_of(L, peer, ctr);
    i32 s_ctr = (i32)__shfl_sync(LB_FULL, L.y, slot < 0 ? 0 : slot);
    if (slot >= 0 && s_ctr == ctr) { uint4 og = p.a_org[ai]; *op = og.x & 0xFFFFu; *oc = (i32)og.y; }
    else { *op = peer; *oc = ctr - 1; }
}

// ---- Fugue sibling scan among the concurrent (future) spans between the cursor and origin_right
// (crdt_rope.rs:101-201).  Uniform serial code on the rare path.
struct SibIn {
    u32 leaf; int from; u32 n_between;
    u32 ol_peer; i32 ol_ctr; u32 or_peer; i32 or_ctr;
    bool pr_valid; u32 pr_leaf; int pr_slot;
    u64 my_peer_id;
};
struct SibOut { bool after_valid; u32 after_peer; i32 after_ctr; };
__device__ __noinline__ SibOut sibling_scan(const SeqPools& p, SibIn in) {
    SeqSmem* sm = seq_sm();
    SibOut out;
    out.after_valid = false;
    out.after_peer = 0;
    out.after_ctr = 0;
    u32 ol_peer = in.ol_peer, or_peer = in.or_peer;
    i32 ol_ctr = in.ol_ctr, or_ctr = in.or_ctr;
    // right parent of the new span: origin_right counts only if its origin_left equals ours
    bool pr_valid = in.pr_valid;
    u64 pr_key = 0;
    if (pr_valid) {
        u32 e_olp;
        i32 e_olc;
        if (or_peer == PEER_UNKNOWN) { e_olp = PEER_NONE; e_olc = -1; }
        else { uint4 og = p.a_org[atom_index(sm, or_peer, or_ctr)]; e_olp = og.x & 0xFFFFu; e_olc = (i32)og.y; }
        pr_valid = e_olp == ol_peer && (ol_peer == PEER_NONE || e_olc == ol_ctr);
        if (pr_valid) pr_key = order_key(p, sm, in.pr_leaf, in.pr_slot);
    }
    bool scanning = false;
    u64 first_key = 0;
    bool have_first = false;
    u32 l2 = in.leaf;
    int from = in.from;
    u32 seen = 0;
    bool stop = false;
    while (l2 != LEAF_NONE && seen < in.n_between && !stop) {
        uint4 S = leaf_load(p, sm, l2);
        int n = leaf_count(S);
        u32 next = __shfl_sync(LB_FULL, S.w, 1);
        for (int s = from; s < n && seen < in.n_between && !stop; s++) {
            u32 o_peer = __shfl_sync(LB_FULL, S.x, s) & 0xFFFFu;
            i32 o_ctr = (i32)__shfl_sync(LB_FULL, S.y, s);
            seen++;
            u64 o_key = order_key(p, sm, l2, s);
            if (!have_first) { first_key = o_key; have_first = true; }
            uint4 oo = p.a_org[atom_index(sm, o_peer, o_ctr)];
            u32 o_olp = oo.x & 0xFFFFu, o_orp = oo.x >> 16;
            i32 o_olc = (i32)oo.y, o_orc = (i32)oo.z;
            bool same_ol = o_olp == ol_peer && (ol_peer == PEER_NONE || o_olc == ol_ctr);
            if (!same_ol) {
                // "visited" is a prefix of the in-between spans: membership is a position test
                bool in_visited = false;
                if (o_olp != PEER_NONE && o_olp != PEER_UNKNOWN && p.atom_leaf[atom_index(sm, o_olp, o_olc)] != LEAF_NONE) {
                    u64 lk = order_key_of_atom(p, sm, o_olp, o_olc);
                    in_visited = lk >= first_key && lk < o_key;
                }
                if (!in_visited) { stop = true; break; }
            }
            if (same_ol) {
                bool same_or = o_orp == or_peer && (or_peer == PEER_NONE || o_orc == or_ctr);
                u64 o_peer_id = sm->dpeer[o_peer].id;
                if (same_or) {
                    if (o_peer_id > in.my_peer_id) { stop = true; break; }
                    scanning = false;
                } else {
                    bool o_pr = false;
                    u64 o_pr_key = 0;
                    if (o_orp != PEER_NONE) {
                        u32 e_olp;
                        i32 e_olc;
                        atom_origin_left(p, sm, o_orp, o_orc, &e_olp, &e_olc);
                        if (e_olp == ol_peer && (ol_peer == PEER_NONE || e_olc == ol_ctr)) {
                            o_pr = true;
                            o_pr_key = order_key_of_atom(p, sm, o_orp, o_orc);
                        }
                    }
                    int cmp;
                    if (o_pr && pr_valid) cmp = o_pr_key < pr_key ? -1 : (o_pr_key > pr_key ? 1 : 0);
                    else if (o_pr) cmp = -1;
                    else if (pr_valid) cmp = 1;
                    else cmp = 0;
                    if (cmp < 0) scanning = true;
                    else if (cmp == 0 && o_peer_id > in.my_peer_id) { stop = true; break; }
                    else scanning = false;
                }
            }
            if (!scanning) { out.after_valid = true; out.after_peer = o_peer; out.after_ctr = o_ctr; }
        }
        l2 = next;
        from = 0;
    }
    return out;
}

// ---- CrdtRope::insert (crdt_rope.rs:43-227)
__device__ __forceinline__ void seq_insert(const SeqPools& p, SeqSmem* sm, u32 peer, i32 ctr, i32 len, i32 pos) {
    int lane = seq_lane();
    for (int attempt = 0; attempt < 4; attempt++) {
        // 1. cursor: right after the pos-th visible atom (prefer-left)
        u32 leaf = sm->first_leaf;
        i32 rem = pos;
        u32 my_link = NODE_NONE;   // lane l remembers the (node, index) the descent took at level l
        bool have_path = false;
        if (pos > 0) {
            u32 nd = sm->root;
            u32 height = sm->height;
            for (u32 lvl = height; lvl >= 1; lvl--) {
                uint2 e = nd_get(p, sm, nd, lane);
                i32 v = (i32)e.y;
                i32 incl = warp_incl_scan(v, lane);
                unsigned m = __ballot_sync(LB_FULL, e.x != NODE_NONE && incl >= rem);
                int idx = __ffs(m) - 1;
                if (idx < 0) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }
                if ((u32)lane == lvl) my_link = (nd << 5) | (u32)idx;
                rem -= __shfl_sync(LB_FULL, incl - v, idx);
                nd = __shfl_sync(LB_FULL, e.x, idx);
            }
            leaf = nd;
            have_path = height < 32;
        }
        uint4 L = leaf_load(p, sm, leaf);
        int n = leaf_count(L);
        int slot = 0;
        i32 off = 0;
        u32 ol_peer = PEER_NONE;
        i32 ol_ctr = -1;
        u32 cur_x = 0;
        i32 cur_ctr = 0, cur_len = 0;
        if (pos > 0) {
            i32 v = s_vis(L);
            i32 incl = warp_incl_scan(v, lane);
            unsigned m = __ballot_sync(LB_FULL, incl >= rem && v > 0);
            slot = __ffs(m) - 1;
            if (slot < 0) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }
            off = rem - __shfl_sync(LB_FULL, incl - v, slot);
            cur_x = __shfl_sync(LB_FULL, L.x, slot);
            cur_ctr = (i32)__shfl_sync(LB_FULL, L.y, slot);
            cur_len = (i32)__shfl_sync(LB_FULL, L.z, slot);
            if ((cur_x & 0xFFFFu) == PEER_UNKNOWN) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }  // beyond the content
            ol_peer = cur_x & 0xFFFFu;
            ol_ctr = cur_ctr + off - 1;
        }
        u32 cur_peer = cur_x & 0xFFFFu;
        bool mid = pos > 0 && off < cur_len;      // the cursor sits inside a span: that span gets cut
        // 2. origin_right: first non-future span at/after the cursor; skipped spans are "in between"
        u32 or_peer = PEER_NONE;
        i32 or_ctr = -1;
        bool pr_valid = false;
        u32 pr_leaf = 0;
        int pr_slot = 0;
        u32 n_between = 0;
        int scan_from = pos > 0 ? slot + 1 : 0;
        if (mid) {
            or_peer = cur_peer;
            or_ctr = cur_ctr + off;
        } else {
            u32 l2 = leaf;
            int from = scan_from;
            uint4 S = L;
            while (true) {
                bool cand = lane >= from && s_peer(S) != PEER_NONE;
                unsigned nonfut = __ballot_sync(LB_FULL, cand && !(S.x & (ST_FUTURE << 16)));
                unsigned fut = __ballot_sync(LB_FULL, cand && (S.x & (ST_FUTURE << 16)));
                if (nonfut) {
                    int f = __ffs(nonfut) - 1;
                    n_between += __popc(fut & ((1u << f) - 1));
                    or_peer = __shfl_sync(LB_FULL, S.x, f) & 0xFFFFu;
                    or_ctr = (i32)__shfl_sync(LB_FULL, S.y, f);
                    pr_leaf = l2;
                    pr_slot = f;
                    pr_valid = true;   // provisional: confirmed by the sibling scan only when needed
                    break;
                }
                n_between += __popc(fut);
                l2 = __shfl_sync(LB_FULL, S.w, 1);
                if (l2 == LEAF_NONE) break;
                from = 0;
                S = leaf_load(p, sm, l2);
            }
        }
        // 3. where to put it
        u32 tgt_leaf = leaf;
        int at = pos > 0 ? slot + 1 : 0;
        if (n_between) {
            SibIn in;
            in.leaf = leaf; in.from = scan_from; in.n_between = n_between;
            in.ol_peer = ol_peer; in.ol_ctr = ol_ctr; in.or_peer = or_peer; in.or_ctr = or_ctr;
            in.pr_valid = pr_valid; in.pr_leaf = pr_leaf; in.pr_slot = pr_slot;
            in.my_peer_id = sm->dpeer[peer].id;
            SibOut so = sibling_scan(p, in);
            if (so.after_valid) {
                tgt_leaf = p.atom_leaf[atom_index(sm, so.after_peer, so.after_ctr)];
                if (tgt_leaf != leaf) { L = leaf_load(p, sm, tgt_leaf); n = leaf_count(L); }
                at = slot_of(L, so.after_peer, so.after_ctr) + 1;
                if (at <= 0) { seq_fail(sm, LB_ERR(DOC_ERR_CORRUPT)); return; }
                mid = false;
            }
        }
        // 4. physical insertion into the loaded image: one new slot, two when the cursor span is cut
        int need = mid ? 2 : 1;
        if (n + need > 32) {
            leaf_split(p, tgt_leaf);
            if (sm->err) return;
            continue;   // positions moved: locate the cursor again
        }
        uint4 og = mk4(0, 0, 0, 0);
        if (mid) og = p.a_org[atom_index(sm, cur_peer, cur_ctr)];   // right origin inherited by the cut-off tail
        u32 link = __shfl_sync(LB_FULL, L.w, 0);
        u32 ux = __shfl_up_sync(LB_FULL, L.x, need);
        u32 uy = __shfl_up_sync(LB_FULL, L.y, need);
        u32 uz = __shfl_up_sync(LB_FULL, L.z, need);
        if (lane >= at + need) { L.x = ux; L.y = uy; L.z = uz; }
        if (lane == at) { L.x = peer; L.y = (u32)ctr; L.z = (u32)len; }
        if (mid) {
            if (lane == at - 1) L.z = (u32)off;
            if (lane == at + 1) { L.x = cur_x; L.y = (u32)(cur_ctr + off); L.z = (u32)(cur_len - off); }
        }
        leaf_store(p, sm, tgt_leaf, L, at > 0 ? at - 1 : 0);
        u64 a0 = atom_index(sm, peer, ctr);
        if (lane == 0) p.a_org[a0] = mk4(ol_peer | (or_peer << 16), (u32)ol_ctr, (u32)or_ctr, 0);
        if (mid && lane == 1)
            p.a_org[atom_index(sm, cur_peer, cur_ctr + off)] = mk4(cur_peer | (og.x & 0xFFFF0000u), (u32)(cur_ctr + off - 1), og.z, 0);
        if (lane < len) p.atom_leaf[a0 + lane] = tgt_leaf;
        for (i32 i = 32 + lane; i < len; i += 32) p.atom_leaf[a0 + i] = tgt_leaf;
        if (have_path && tgt_leaf == leaf) {   // every level of the recorded path at once
            if (my_link != NODE_NONE) nd_add_vis(p, sm, my_link >> 5, (int)(my_link & 31), len);
            __syncwarp();
        } else add_vis(p, sm, link, len);
        return;
    }
    seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY));
}

// ---- container switching: internal nodes < NS and the tracker version live in shared memory while a
// container is active
__device__ __noinline__ void store_container(const SeqPools& p, const BatchTables& t, u64 cid0, u32 cidx) {
    if (cidx == 0xFFFFFFFFu) return;
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    __syncwarp();
    u32 cached = sm->n_nodes < LB_SEQ_NS ? sm->n_nodes : LB_SEQ_NS;
    for (u32 nd = 0; nd < cached; nd++) {
        p.node[(sm->node0 + nd) * 32 + lane] = mk2(sm->child[nd][lane], (u32)sm->vis[nd][lane]);
        if (lane == 0) p.node_parent[sm->node0 + nd] = sm->parent[nd];
    }
    if ((u32)lane < sm->P) p.cvv[sm->cvv0 + lane] = sm->cvv[lane];
#ifdef LB_SIMT_EMU
    if (lane == 0 && getenv("LB_EMU_STATS")) fprintf(stderr, "container %u: leaves %u nodes %u height %u root %u\n", cidx, sm->n_leaves, sm->n_nodes, sm->height, sm->root);
#endif
    if (lane == 0) {
        DocContainer& dc = t.dcont[cid0 + cidx];
        dc.n_leaves = sm->n_leaves;
        dc.n_nodes = sm->n_nodes;
        dc.root = sm->root;
        dc.height = sm->height;
        dc.first_leaf = sm->first_leaf;
        dc.unk_sid = sm->unk_leaf;
    }
    __syncwarp();
}
// Tracker::new_with_unknown (tracker.rs:38-63) on first use: one placeholder span of length u32::MAX/4
__device__ __noinline__ void load_container(const SeqPools& p, const BatchTables& t, u64 cid0, u32 cidx) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    const DocContainer& dc = t.dcont[cid0 + cidx];
    const u64 leaf0 = dc.leaf0, node0 = dc.node0, cvv0 = dc.cvv0;
    u32 n_leaves = dc.n_leaves, n_nodes = dc.n_nodes;
    __syncwarp();
    if (lane == 0) {
        sm->leaf0 = leaf0;
        sm->node0 = node0;
        sm->cvv0 = cvv0;
        sm->leaf_cap = dc.leaf_cap;
        sm->node_cap = dc.node_cap;
        sm->n_leaves = n_leaves;
        sm->n_nodes = n_nodes;
        sm->root = dc.root;
        sm->height = dc.height;
        sm->first_leaf = dc.first_leaf;
        sm->unk_leaf = dc.unk_sid;
    }
    if (n_leaves == 0) {
        if (dc.leaf_cap < 1 || dc.node_cap < 1) { seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY)); return; }
        if (lane == 0) {
            sm->n_leaves = 1;
            sm->n_nodes = 1;
            sm->root = 0;
            sm->height = 1;
            sm->first_leaf = 0;
            sm->unk_leaf = 0;
        }
        // leaf 0: the placeholder span; parent link (node 0, index 0) in slot 0, no next leaf in slot 1
        p.leaf[leaf0 * 32 + lane] = mk4(lane == 0 ? (u32)PEER_UNKNOWN : SLOT_EMPTY, 0, lane == 0 ? (u32)UNKNOWN_LEN : 0u,
                                        lane == 1 ? LEAF_NONE : 0u);
        nd_set(p, sm, 0, lane, lane == 0 ? 0u : NODE_NONE, lane == 0 ? (i32)UNKNOWN_LEN : 0);
        if (lane == 0) nd_set_parent(p, sm, 0, NODE_NONE);
        sm->cvv[lane] = 0;
        for (u32 q = 32 + (u32)lane; q < sm->P; q += 32) p.cvv[cvv0 + q] = 0;
        __syncwarp();
        return;
    }
    u32 cached = n_nodes < LB_SEQ_NS ? n_nodes : LB_SEQ_NS;
    for (u32 nd = 0; nd < cached; nd++) {
        uint2 e = p.node[(node0 + nd) * 32 + lane];
        sm->child[nd][lane] = e.x;
        sm->vis[nd][lane] = (i32)e.y;
        if (lane == 0) sm->parent[nd] = p.node_parent[node0 + nd];
    }
    sm->cvv[lane] = (u32)lane < sm->P ? p.cvv[cvv0 + lane] : 0;
    __syncwarp();
}

// ---- emit the final visible runs of the active container (after checkout to the final version)
__device__ __noinline__ void emit_output(const SeqPools& p, const BatchTables& t, u64 cid0, u32 cidx) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    DocContainer& dc = t.dcont[cid0 + cidx];
    u32 n_out = 0;
    u32 total = 0;
    u32 l2 = sm->first_leaf;
    u32 out_cap = dc.out_cap;
    u64 out0 = dc.out0;
    while (l2 != LEAF_NONE) {
        uint4 L = leaf_load(p, sm, l2);
        u32 pe = s_peer(L);
        bool live = pe != PEER_NONE && pe != PEER_UNKNOWN && s_st(L) == 0;
        unsigned m = __ballot_sync(LB_FULL, live);
        if (live) {
            u32 o = n_out + __popc(m & ((1u << lane) - 1));
            if (o < out_cap) {
                u32 row = t.atom_row[atom_index(sm, pe, (i32)L.y)];
                t.out_row[out0 + o] = row;
                t.out_off[out0 + o] = (u32)((i32)L.y - t.op_counter[row]);
                t.out_len[out0 + o] = L.z;
            }
        }
        total += (u32)warp_sum(live ? (i32)L.z : 0);
        n_out += __popc(m);
        l2 = __shfl_sync(LB_FULL, L.w, 1);
    }
    if (n_out > out_cap) seq_fail(sm, LB_ERR(DOC_ERR_CAPACITY));
    __syncwarp();
    if (lane == 0) {
        dc.n_out = n_out < out_cap ? n_out : out_cap;
        dc.seq_len = total;
    }
    __syncwarp();
}

// (single-peer documents do not skip the origin records, although nothing is ever concurrent in them: such a flag costs
//  a register in every helper of a kernel that spills at its register budget)
// One document by one warp.  Every per-document field of `sm` (err, abase, the active container, cvv) is set again
// here before it is read: the warp's previous document left its values there.
__device__ __forceinline__ void integrate_doc(DocInfo& di, SeqSmem* sm, int lane, const SeqPools& pools, const BatchTables& tables) {
    if (di.code != DOC_OK || di.n_applied == 0) return;
    const u64 cid0 = di.cid0, ch0 = di.ch0, vv0 = di.vv0;
    const u32 P = di.P, C = di.C, n_applied = di.n_applied;
    bool any = false;
    for (u32 ci = 0; ci < C; ci++)
        if (tables.dcont[cid0 + ci].leaf_cap) any = true;
    if (!any) return;
    const DocPeer* dpeer = tables.dpeer + di.peer0;
    sm->abase[lane] = (u32)lane < P ? dpeer[lane].atom_base : 0;
    if (lane == 0) {
        sm->dpeer = dpeer;
        sm->atom0 = di.atom0;
        sm->P = P;
        sm->err = 0;
    }
    __syncwarp();
    for (u32 ci = lane; ci < C; ci += 32) pools.cont_epoch[cid0 + ci] = 0xFFFFFFFFu;
    __syncwarp();
    u32 cidx = 0xFFFFFFFFu;
    u32 prev_peer = 0xFFFFFFFFu;
    u32 cur_epoch = 0xFFFFFFFFu;   // epoch of the active container (register; spilled on container switch)
    for (u32 kb = 0; kb < n_applied && !sm->err; kb += 32) {
        // ---- 32 change headers of the walk per round trip
        u32 kk = kb + (u32)lane;
        u32 h_ch = 0, h_peer = 0, h_r0 = 0, h_nr = 0, h_pos = 0;
        bool h_simple = false;
        if (kk < n_applied) {
            h_ch = tables.ch_walk[ch0 + kk];
            h_peer = tables.ch_peer[h_ch];
            h_r0 = (u32)tables.ch_op0[h_ch];
            h_nr = tables.ch_nops[h_ch];
            h_pos = tables.ch_pos[h_ch];
            h_simple = tables.ch_dep_self[h_ch] && tables.ch_ndeps[h_ch] == 0;
        }
        u32 cnt = n_applied - kb < 32 ? n_applied - kb : 32;
        for (u32 j = 0; j < cnt && !sm->err; j++) {
            u32 k = kb + j;
            u32 peer = __shfl_sync(LB_FULL, h_peer, j);
            u32 r0 = __shfl_sync(LB_FULL, h_r0, j);
            u32 nr = __shfl_sync(LB_FULL, h_nr, j);
            u32 pos = __shfl_sync(LB_FULL, h_pos, j);
            // fast path (no checkout): the change only depends on its predecessor, which was the previous change
            // of the walk, and the container's tracker sat at that version when it was last touched
            bool chain = __shfl_sync(LB_FULL, (int)h_simple, j) && prev_peer == peer && k > 0;
            const i32* vv = tables.ch_vv + vv0 + (u64)pos * P;
            i32 cvv_dirty = -1;   // end counter of this change's last op in the active container, not yet in cvv
            for (u32 rb = 0; rb < nr && !sm->err; rb += 32) {
                // ---- 32 op records per round trip
                uint4 rec = mk4(0, 0, 0, 0);
                u32 aux = 0;
                if (rb + (u32)lane < nr) { rec = tables.op_rec[r0 + rb + lane]; aux = tables.op_aux[r0 + rb + lane]; }
                u32 kind_l = REC_KIND(rec.x);
                // deletes: (possibly stale) home leaf of the first target atom
                u32 hint_l = kind_l == OPK_SEQ_DEL ? pools.atom_leaf[atom_index(sm, aux, (i32)rec.w)] : LEAF_NONE;
                unsigned m = __ballot_sync(LB_FULL, kind_l == OPK_SEQ_INS || kind_l == OPK_SEQ_DEL);
                while (m && !sm->err) {
                    int s = __ffs(m) - 1;
                    m &= m - 1;
                    u32 rx = __shfl_sync(LB_FULL, rec.x, s);
                    i32 ctr = (i32)__shfl_sync(LB_FULL, rec.y, s);
                    i32 len = (i32)__shfl_sync(LB_FULL, rec.z, s);
                    i32 prop = (i32)__shfl_sync(LB_FULL, rec.w, s);
                    u32 ci = REC_CIDX(rx);
                    if (ci != cidx) {
                        if (cidx != 0xFFFFFFFFu && lane == 0) pools.cont_epoch[cid0 + cidx] = cur_epoch;
                        if (cvv_dirty >= 0) { __syncwarp(); if (lane == 0) cvv_set(pools, sm, peer, cvv_dirty); cvv_dirty = -1; }
                        store_container(pools, tables, cid0, cidx);
                        load_container(pools, tables, cid0, ci);
                        cidx = ci;
                        if (sm->err) break;
                        cur_epoch = pools.cont_epoch[cid0 + ci];
                    }
                    if (cur_epoch != k) {
                        if (!(chain && cur_epoch == k - 1)) checkout(pools, tables, sm, ch0, cidx, vv, peer, ctr);
                        cur_epoch = k;
                    }
                    if (REC_KIND(rx) == OPK_SEQ_INS) seq_insert(pools, sm, peer, ctr, len, prop);
                    else   // delete by target id (crdt_rope.rs:236-315 ; tracker.rs:173-232)
                        range_apply(pools, __shfl_sync(LB_FULL, aux, s), prop, prop + len, -1, +1, __shfl_sync(LB_FULL, hint_l, s));
                    // current_vv of the tracker follows its own ops (tracker.rs:131-139, 228-231); in causal order
                    // this entry only grows: written back when the container or the change ends
                    cvv_dirty = ctr + len;
                }
            }
            if (cvv_dirty >= 0) { __syncwarp(); if (lane == 0) cvv_set(pools, sm, peer, cvv_dirty); __syncwarp(); }
            prev_peer = peer;
        }
    }
    // final version = everything applied, or the requested version of a checkout (k_checkout.cuh): the atoms past it were
    // never integrated, and their atom -> row entries were never written
    for (u32 ci = 0; ci < C && !sm->err; ci++) {
        const DocContainer& dc = tables.dcont[cid0 + ci];
        if (!dc.leaf_cap || (dc.n_leaves == 0 && ci != cidx)) continue;
        if (ci != cidx) {
            store_container(pools, tables, cid0, cidx);
            load_container(pools, tables, cid0, ci);
            cidx = ci;
        }
        for (u32 q = 0; q < P && !sm->err; q++) {
            i32 tgt = tables.ck_end ? tables.ck_end[(sm->dpeer - tables.dpeer) + q] : sm->dpeer[q].end_counter;
            i32 cur = cvv_get(pools, sm, q);
            if (cur > tgt) toggle_ops(pools, tables, ch0, cidx, q, tgt, cur, -1);
            else if (cur < tgt) toggle_ops(pools, tables, ch0, cidx, q, cur, tgt, +1);
            __syncwarp();
            if (lane == 0) cvv_set(pools, sm, q, tgt);
            __syncwarp();
        }
        if (!sm->err) emit_output(pools, tables, cid0, cidx);
    }
    store_container(pools, tables, cid0, cidx);
    __syncwarp();
    if (lane == 0 && sm->err) di.code = sm->err;
}

// QUEUE = 1, for batches with more documents than the device holds warps: the launch holds only as many CTAs as can be
// resident at once (engine.cu), and every warp takes the next document from `pools.next_doc` until none are left.  A
// warp whose document ends early starts another instead of holding its slot until the slowest warp of its CTA is done,
// and no last wave of CTAs runs half full.  QUEUE = 0: warp w of the grid integrates document w; with every document
// on a warp of its own the queue has nothing to balance, and its loop made the one-document C4 0.8 % slower (at 8 CTAs
// per SM, DESIGN.md section 6).
// 8 CTAs x 4 warps = 32 resident documents per SM (64 registers/thread).  With the warp-uniform context in shared
// memory the kernel spills little enough that more documents in flight win: on H100, C3 integrates fastest at 8 of the
// 4, 5, 6, 8 and 10 measured (DESIGN.md section 3).
#define LB_SEQ_MINB 8
template <int QUEUE>
__global__ void __launch_bounds__(32 * LB_SEQ_WARPS, LB_SEQ_MINB)
k_seq_integrate(DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ SeqPools pools,
                const __grid_constant__ BatchTables tables) {
    SeqSmem* sm = seq_sm();
    int lane = seq_lane();
    if (!QUEUE) {
        u32 d = blockIdx.x * LB_SEQ_WARPS + (threadIdx.x >> 5);
        if (d < n_docs) integrate_doc(docs[d], sm, lane, pools, tables);
        return;
    }
    while (true) {
        u32 d = 0;
        if (lane == 0) d = atomicAdd(pools.next_doc, 1u);
        d = __shfl_sync(LB_FULL, d, 0);
        if (d >= n_docs) return;
        integrate_doc(docs[d], sm, lane, pools, tables);
    }
}
