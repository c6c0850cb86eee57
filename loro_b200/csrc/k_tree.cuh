// loro_b200 -- phase 5b: movable tree (one warp per document).
//
// Replaces (reference, relative to crates/loro-internal/src):
//   diff_calc/tree.rs:21-148 (TreeDiffCalculator: ops of a tree in (lamport, peer) order), :417-452
//     (MoveLamportAndID ordering), :471-508 (TreeCacheForDiff::apply / is_ancestor_of: a move whose new parent is
//     a descendant of the target is recorded but not effected)
//   state/tree_state.rs:690-747 (TreeState::mov with the cycle check, used for imports into a fresh document),
//     :592-595 + :61-67 (children ordered by (fractional index bytes, lamport, peer) = NodePosition),
//     :749-760 (is_node_deleted: a node is alive iff its parent chain reaches the root)
//   loro-common/src/lib.rs:631 (DELETED_TREE_ROOT: a delete is a move under it)
//
// Shape: a tree's ops are totally ordered by (lamport, peer) and every op depends on the tree the earlier ones
// left, so the apply is sequential per tree; the parallelism is across documents (config C5: 10^4 of them).
// Everything around the sequential core is lane-parallel: the document's RawTreeMove records are sorted by a
// 64-bit key with a warp bitonic network over global memory (the records are L2-resident), 32 records are fetched
// per round trip, and the sibling lists come out of a second sort of the nodes by (parent slot, position prefix)
// with the full NodePosition comparison as tie-break.  Node tables are dense arrays over the document's atoms
// (a TreeID is the id of its create op), so "node -> parent" is one load.
// Nodes of different tree containers share the atom-indexed tables: in a well-formed document their ids are
// disjoint; a hostile blob that moves a node of one tree inside another gets a memory-safe, cycle-free result.
#pragma once
#include "lb_tables.cuh"

__device__ __forceinline__ u32* tree_sub(const BatchTables& t, const DocInfo& di) { return (u32*)(t.ns_key + di.tree0); }

// decimal digits of v: compare against powers of ten around the estimate from the bit length (no 64-bit divisions)
__device__ const u64 LB_P10[20] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull, 1000000000ull,
                         10000000000ull, 100000000000ull, 1000000000000ull, 10000000000000ull, 100000000000000ull,
                         1000000000000000ull, 10000000000000000ull, 100000000000000000ull, 1000000000000000000ull,
                         10000000000000000000ull};
__device__ __forceinline__ u32 dec_digits(u64 v) {
    if (v == 0) return 1;
    u32 bits = 64u - (u32)__clzll((long long)v);
    u32 k = (bits * 1233u) >> 12;          // floor(log10(2^bits)) : k or k + 1 digits
    return k + (v >= LB_P10[k] ? 1u : 0u);
}
// "<counter>@<peer>" with its quotes
__device__ inline u32 tree_id_len(const DocPeer* dpeer, u32 P, u32 a) {
    u32 p = 0;
    for (u32 q = 0; q < P; q++)
        if (a >= dpeer[q].atom_base && a < dpeer[q].atom_base + (u32)dpeer[q].end_counter) { p = q; break; }
    return 3 + dec_digits(a - dpeer[p].atom_base) + dec_digits(dpeer[p].id);
}
// bytes of a node's object before / after its children when its meta map is empty (keys in ascending order):
//   [,]{"children":[   ...   ],"fractional_index":"HEX","id":"c@p","index":N,"meta":{},"parent":null|"c@p"}
__device__ __forceinline__ u32 tree_open_len(u32 sib) { return 13u + (sib ? 1u : 0u); }
__device__ inline u32 tree_close_len(const DocPeer* dpeer, u32 P, u32 node, u32 parent, u32 sib, u32 pos_len) {
    return 1 + 21 + 2 * pos_len + 7 + tree_id_len(dpeer, P, node) + 9 + dec_digits(sib) + 10 + 10 +
           (parent == TREE_ROOT ? 4u : tree_id_len(dpeer, P, parent)) + 1;
}

// ---- warp bitonic sort of (key, val) pairs in global memory, any n (partners beyond n act as +inf: with every
// comparator pointing the same way they never have to move).  `tie(a, b)` orders two vals whose keys are equal.
template <class Tie>
__device__ inline void warp_sort_pairs(u64* key, u32* val, u32 n, int lane, Tie tie) {
    if (n < 2) return;
    for (u32 k = 2; (k >> 1) < n; k <<= 1) {
        for (u32 j = k >> 1; j > 0; j >>= 1) {
            bool flip = j == (k >> 1);
            for (u32 i = (u32)lane; i < n; i += 32) {
                u32 l = flip ? (i ^ (k - 1)) : (i ^ j);
                if (l > i && l < n) {
                    u64 ki = key[i], kl = key[l];
                    bool sw = ki > kl;
                    u32 vi = val[i], vl = val[l];
                    if (ki == kl && ki != ~0ull) sw = tie(vl, vi);   // +inf entries carry no payload to compare
                    if (sw) { key[i] = kl; key[l] = ki; val[i] = vl; val[l] = vi; }
                }
            }
            __syncwarp();
        }
    }
}
struct NoTie { __device__ bool operator()(u32, u32) const { return false; } };
// same network on values only, ordered by `before(a, b)`
template <class Before>
__device__ inline void warp_sort_vals(u32* val, u32 n, int lane, Before before) {
    if (n < 2) return;
    for (u32 k = 2; (k >> 1) < n; k <<= 1) {
        for (u32 j = k >> 1; j > 0; j >>= 1) {
            bool flip = j == (k >> 1);
            for (u32 i = (u32)lane; i < n; i += 32) {
                u32 l = flip ? (i ^ (k - 1)) : (i ^ j);
                if (l > i && l < n) {
                    u32 vi = val[i], vl = val[l];
                    if (before(vl, vi)) { val[i] = vl; val[l] = vi; }
                }
            }
            __syncwarp();
        }
    }
}

// lexicographic comparison of two fractional indexes (FractionalIndex derives Ord on its bytes)
__device__ inline int pos_cmp(const BatchTables& t, u32 pa, u32 pb) {
    if (pa == pb) return 0;
    const u8* a = t.pos_pool + t.pos_off[pa];
    const u8* b = t.pos_pool + t.pos_off[pb];
    u32 la = t.pos_len[pa], lb = t.pos_len[pb];
    u32 n = la < lb ? la : lb;
    for (u32 i = 0; i < n; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

// Three kernels, one warp per document each:
//   k_tree_sort    the document's tree ops in (lamport, peer) order (counting sort on global scratch)
//   k_tree_apply   the sequential apply -- ONE chain of dependent parent look-ups per warp, so the links live in shared
//                  memory (16-bit, documents with fewer than TREE_S_NODES atoms) and few warps per SM are enough
//   k_tree_layout  sibling lists and the JSON layout: lane-parallel walks, best at full occupancy, links from global
// (one kernel holding the shared-memory links through all three steps was measured: the low occupancy it forces on the
//  lane-parallel steps cost more than the fast links gained -- 119 ms instead of 65 ms on config C5.)
#define TREE_WARPS 1          // one document per CTA: the shared-memory size per document decides how many are resident
#define TREE_S_NODES_MAX 32768 // larger documents keep their links in global memory
struct ParentArr {
    u16* s;      // nullptr: global only
    u32* g;
    __device__ __forceinline__ u32 get(u32 i) const {
        if (!s) return g[i];
        u16 v = s[i];
        return v >= 0xFFFDu ? 0xFFFF0000u | v : (u32)v;
    }
    __device__ __forceinline__ void set(u32 i, u32 v) const { if (s) s[i] = (u16)v; else g[i] = v; }   // (special values keep their low 16 bits)
};

__global__ void k_tree_sort(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t) {
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK || !di.has_tree) return;
    const u32 A = (u32)di.atom_total, C = di.C;
    const u64 base = di.tree0;
    for (u32 i = lane; i < A + C; i += 32) { t.tn_cnt[base + i] = 0; t.tn_base[base + i] = 0; }
    // ---- the document's tree ops (contiguous: blocks of a document are) in (lamport, peer) order.
    // Lamports are recomputed from the dependencies, so they are smaller than the document's atom count: a counting
    // sort over the lamport (tn_cnt / tn_base double as histogram and offsets) followed by a per-lamport fix of the
    // few ties replaces the O(n log^2 n) network; a lamport outside the range falls back to the network.
    const u64 tr_lo = t.blocks[di.b0].tr0, tr_hi = t.blocks[di.b1].tr0;
    const u32 n_tr = (u32)(tr_hi - tr_lo);
    u64* skey = t.ts_key + tr_lo;
    u32* sval = t.ts_val + tr_lo;
    u32* cnt = t.tn_cnt + base;
    u32* off = t.tn_base + base;
    __syncwarp();
    bool wide = false;
    for (u32 i = lane; i < n_tr; i += 32) {
        u64 k = t.tr_key[tr_lo + i];
        if (k == ~0ull) continue;
        u32 lam = (u32)(k >> 32);
        if (lam >= A) wide = true; else atomicAdd(&cnt[lam], 1u);
    }
    wide = __any_sync(LB_FULL, wide);
    if (wide) {
        for (u32 i = lane; i < A; i += 32) cnt[i] = 0;
        for (u32 i = lane; i < n_tr; i += 32) { skey[i] = t.tr_key[tr_lo + i]; sval[i] = i; }
        __syncwarp();
        warp_sort_pairs(skey, sval, n_tr, lane, NoTie());
    } else {
        u32 carry = 0;
        for (u32 i0 = 0; i0 < A; i0 += 32) {
            u32 i = i0 + (u32)lane;
            int c = i < A ? (int)cnt[i] : 0;
            int incl = warp_incl_scan(c, lane);
            if (i < A) off[i] = carry + (u32)(incl - c);
            carry += (u32)__shfl_sync(LB_FULL, incl, 31);
        }
        const u32 n_valid = carry;
        __syncwarp();
        for (u32 i = lane; i < n_tr; i += 32) {
            u64 k = t.tr_key[tr_lo + i];
            if (k == ~0ull) continue;
            u32 lam = (u32)(k >> 32);
            u32 pos = off[lam] + (atomicSub(&cnt[lam], 1u) - 1u);
            skey[pos] = k;
            sval[pos] = i;
        }
        for (u32 i = n_valid + (u32)lane; i < n_tr; i += 32) skey[i] = ~0ull;
        __syncwarp();
        for (u32 lam = lane; lam < A; lam += 32) {   // concurrent ops with the same lamport: order by peer
            u32 b = off[lam], e = lam + 1 < A ? off[lam + 1] : n_valid;
            for (u32 x = b + 1; x < e; x++) {
                u64 kx = skey[x]; u32 vx = sval[x];
                u32 y = x;
                while (y > b && skey[y - 1] > kx) { skey[y] = skey[y - 1]; sval[y] = sval[y - 1]; y--; }
                skey[y] = kx; sval[y] = vx;
            }
        }
    }
    __syncwarp();
    // the records in apply order: the sequential loop of k_tree_apply then reads them with coalesced loads instead of a
    // key -> index -> record chain of three dependent round trips per 32 ops
    for (u32 j = lane; j < n_tr; j += 32) {
        uint4 rec;
        rec.x = rec.y = rec.z = 0; rec.w = 0xFFFFFFFFu;
        if (skey[j] != ~0ull) rec = t.tr_rec[tr_lo + sval[j]];
        t.ts_rec[tr_lo + j] = rec;
    }
}

__global__ void __launch_bounds__(32 * TREE_WARPS) k_tree_apply(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t, u32 s_nodes) {
#ifdef LB_SIMT_EMU
    LB_DYN_SMEM(u16, tree_smem);
#else
    extern __shared__ __align__(16) u16 tree_smem[];
#endif
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK || !di.has_tree) return;
    const u32 A = (u32)di.atom_total;
    const u64 base = di.tree0;
    ParentArr parent;
    parent.g = t.tn_parent + base;
    parent.s = A <= s_nodes ? tree_smem + (threadIdx.x >> 5) * s_nodes : nullptr;
    u32* move = t.tn_move + base;
    for (u32 i = lane; i < A; i += 32) parent.set(i, TREE_UNEXIST);
    const u64 tr_lo = t.blocks[di.b0].tr0, tr_hi = t.blocks[di.b1].tr0;
    const u32 n_tr = (u32)(tr_hi - tr_lo);
    const u32* sval = t.ts_val + tr_lo;
    __syncwarp();
    // ---- sequential apply, 32 records per round trip, the next 32 in flight meanwhile
    const uint4* srec = t.ts_rec + tr_lo;
    bool stop = false;
    uint4 nrec;
    u32 nti = 0;
    nrec.x = nrec.y = nrec.z = 0; nrec.w = 0xFFFFFFFFu;
    if ((u32)lane < n_tr) { nrec = srec[lane]; nti = sval[lane]; }
    for (u32 j0 = 0; j0 < n_tr && !stop; j0 += 32) {
        uint4 rec = nrec;
        u32 ti_l = nti;
        {
            u32 jn = j0 + 32 + (u32)lane;
            nrec.w = 0xFFFFFFFFu;
            if (jn < n_tr) { nrec = srec[jn]; nti = sval[jn]; }
        }
        u32 cnt = n_tr - j0 < 32 ? n_tr - j0 : 32;
        for (u32 s = 0; s < cnt; s++) {
            u32 row = __shfl_sync(LB_FULL, rec.w, (int)s);
            if (row == 0xFFFFFFFFu) { stop = true; break; }   // not applied: these sort last
            u32 target = __shfl_sync(LB_FULL, rec.x, (int)s);
            u32 np = __shfl_sync(LB_FULL, rec.y, (int)s);
            u32 ti = __shfl_sync(LB_FULL, ti_l, (int)s);
            bool effected = true;
            if (np < TREE_UNEXIST && parent.get(target) != TREE_UNEXIST) {
                // is the target an ancestor of (or equal to) the new parent?  (tree.rs:477-508, tree_state.rs:727-747)
                // This walk is the kernel: one dependent look-up per level, so the shared-memory form is kept minimal
                if (parent.s) {
                    const u16* ps = parent.s;
                    u32 cur = np;
                    for (u32 guard = 0; guard <= A; guard++) {
                        if (cur == target) { effected = false; break; }
                        cur = ps[cur];
                        if (cur >= 0xFFFDu) break;   // root / deleted root / no parent yet
                    }
                } else {
                    u32 cur = np;
                    for (u32 guard = 0; guard <= A; guard++) {
                        if (cur == target) { effected = false; break; }
                        u32 pp = parent.g[cur];
                        if (pp >= TREE_UNEXIST) break;
                        cur = pp;
                    }
                }
            }
            __syncwarp();
            if (effected && lane == 0) { parent.set(target, np); move[target] = ti; }
            __syncwarp();
        }
    }
    __syncwarp();
    __syncwarp();
    if (parent.s) for (u32 i = lane; i < A; i += 32) parent.g[i] = parent.get(i);   // the later passes read the global table
}

__global__ void k_tree_layout(DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t) {
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK || !di.has_tree) return;
    const u32 A = (u32)di.atom_total, C = di.C;
    const u64 base = di.tree0;
    const u32* parent = t.tn_parent + base;
    const u32* move = t.tn_move + base;
    u32* cnt = t.tn_cnt + base;
    u32* off = t.tn_base + base;
    const u64 tr_lo = t.blocks[di.b0].tr0, tr_hi = t.blocks[di.b1].tr0;
    // ---- sibling lists: nodes bucketed by parent slot (counting sort), every list ordered by NodePosition =
    // (fractional index bytes, lamport, peer); lists are short (fan-out), so a lane sorts a list by insertion with an
    // 8-byte position prefix as the first comparison; a list longer than 32 goes through the warp network.
    // Every pass below touches a node a constant number of times: the passes that used to climb the parent chain per
    // node (root of the tree, subtree sizes, offsets) made 80 scattered sector reads per node -- with a few GB of
    // node tables resident across the chip they all went to HBM, and they were the kernel's whole time.
    u64* nkey = t.ns_key + base;
    u32* child = t.tn_child + base;
    u32* fill = t.tn_sib + base;
    u32* root = t.tn_root + base;
    u32* slot_tmp = t.tn_aclose + base;   // parent slot of a node until the lists are built
    u32* plen_tmp = t.tn_aopen + base;    // length of the node's fractional index until the offsets are written
    for (u32 i = lane; i < A + C; i += 32) { cnt[i] = 0; fill[i] = 0; }
    __syncwarp();
    for (u32 a = lane; a < A; a += 32) {
        u32 p = parent[a];
        root[a] = TREE_UNEXIST;
        if (p == TREE_UNEXIST || p == TREE_DELETED) { slot_tmp[a] = TREE_UNEXIST; continue; }
        uint4 rec = t.tr_rec[tr_lo + move[a]];
        u32 sl = p == TREE_ROOT ? A + t.op_cidx[rec.w] : p;
        slot_tmp[a] = sl;
        atomicAdd(&cnt[sl], 1u);
        const u8* pb = t.pos_pool + t.pos_off[rec.z];
        u32 pl = t.pos_len[rec.z];
        plen_tmp[a] = pl;
        u64 pre = 0;
        for (u32 k = 0; k < 8; k++) pre = (pre << 8) | (k < pl ? pb[k] : 0u);
        nkey[a] = pre;
    }
    __syncwarp();
    {
        u32 carry = 0;
        for (u32 i0 = 0; i0 < A + C; i0 += 32) {
            u32 i = i0 + (u32)lane;
            int c = i < A + C ? (int)cnt[i] : 0;
            int incl = warp_incl_scan(c, lane);
            if (i < A + C) off[i] = carry + (u32)(incl - c);
            carry += (u32)__shfl_sync(LB_FULL, incl, 31);
        }
    }
    __syncwarp();
    for (u32 a = lane; a < A; a += 32) {
        u32 sl = slot_tmp[a];
        if (sl != TREE_UNEXIST) child[off[sl] + atomicAdd(&fill[sl], 1u)] = a;
    }
    __syncwarp();
    auto before = [&](u32 a, u32 b) -> bool {   // NodePosition order (tree_state.rs:61-67)
        u64 ka = nkey[a], kb = nkey[b];
        if (ka != kb) return ka < kb;
        uint4 ra = t.tr_rec[tr_lo + move[a]], rb = t.tr_rec[tr_lo + move[b]];
        int c = pos_cmp(t, ra.z, rb.z);
        if (c) return c < 0;
        return t.tr_key[tr_lo + move[a]] < t.tr_key[tr_lo + move[b]];
    };
    bool big = false;
    for (u32 sl = lane; sl < A + C; sl += 32) {
        u32 n = cnt[sl], b0 = off[sl];
        if (n > 32) { big = true; continue; }
        for (u32 x = 1; x < n; x++) {
            u32 vx = child[b0 + x], y = x;
            while (y > 0 && before(vx, child[b0 + y - 1])) { child[b0 + y] = child[b0 + y - 1]; y--; }
            child[b0 + y] = vx;
        }
    }
    if (__any_sync(LB_FULL, big)) {
        for (u32 s0 = 0; s0 < A + C; s0 += 32) {
            u32 sl = s0 + (u32)lane;
            unsigned m = __ballot_sync(LB_FULL, sl < A + C && cnt[sl] > 32);
            while (m) {
                int q = __ffs(m) - 1;
                m &= m - 1;
                u32 bs = s0 + (u32)q;
                warp_sort_vals(child + off[bs], cnt[bs], lane, before);
            }
        }
    }
    __syncwarp();
    for (u32 sl = lane; sl < A + C; sl += 32) {
        u32 n = cnt[sl], b0 = off[sl];
        for (u32 x = 0; x < n; x++) t.tn_sib[base + child[b0 + x]] = x;
    }
    __syncwarp();
    // ---- JSON layout of the hierarchy (meta maps assumed empty; a document where a node's meta map exists keeps
    // the serial walk).  The sort keys are dead: their space becomes sub[] / rel[].
    const DocPeer* dpeer = t.dpeer + di.peer0;
    const u32 P = di.P;
    bool has_meta = false;
    for (u32 c = lane; c < C; c += 32) {
        const DocContainer& dc = t.dcont[di.cid0 + c];
        if (dc.is_root || dc.type != CT_MAP || dc.key_or_peer >= P) continue;
        const DocPeer& dp = dpeer[dc.key_or_peer];
        if (dc.counter >= 0 && dc.counter < dp.end_counter && parent[dp.atom_base + (u32)dc.counter] != TREE_UNEXIST) has_meta = true;
    }
    has_meta = __any_sync(LB_FULL, has_meta);
    u32* sub = (u32*)nkey;
    u32* rel = sub + (A + C);
    // alive nodes level by level (breadth first from the root slots; the children of a node stay adjacent and in
    // sibling order): order[] / lvl[] live in the sort space of k_tree_sort, which the apply has finished with --
    // a node has a create op, so there are at most n_tr nodes and n_tr levels
    u32* order = t.ts_val + tr_lo;
    u32* lvl = (u32*)(t.ts_key + tr_lo);
    const u32 n_tr = (u32)(tr_hi - tr_lo);
    u32 n_lvl = 0, lo = 0, hi = 0;
    {   // level 0: the children of every root slot
        u32 carry = 0;
        for (u32 c0 = 0; c0 < C; c0 += 32) {
            u32 c = c0 + (u32)lane;
            u32 n = c < C ? cnt[A + c] : 0u;
            int incl = warp_incl_scan((int)n, lane);
            u32 w = carry + (u32)incl - n;
            if (n) { u32 b0 = off[A + c]; for (u32 k = 0; k < n; k++) { u32 x = child[b0 + k]; order[w + k] = x; root[x] = A + c; } }
            carry += (u32)__shfl_sync(LB_FULL, incl, 31);
        }
        hi = carry;
    }
    __syncwarp();
    while (hi > lo && n_lvl + 1 < 2 * n_tr) {
        if (lane == 0) lvl[n_lvl] = lo;
        n_lvl++;
        u32 carry = hi;
        for (u32 i0 = lo; i0 < hi; i0 += 32) {
            u32 i = i0 + (u32)lane;
            u32 p = i < hi ? order[i] : 0u;
            u32 n = i < hi ? cnt[p] : 0u;
            int incl = warp_incl_scan((int)n, lane);
            u32 w = carry + (u32)incl - n;
            if (n) { u32 b0 = off[p], r = root[p]; for (u32 k = 0; k < n; k++) { u32 x = child[b0 + k]; order[w + k] = x; root[x] = r; } }
            carry += (u32)__shfl_sync(LB_FULL, incl, 31);
        }
        lo = hi;
        hi = carry;
        __syncwarp();
    }
    if (lane == 0) lvl[n_lvl] = lo;   // == number of alive nodes
    __syncwarp();
    // bottom-up: JSON bytes of every subtree, offset of every child inside its parent's children list
    for (u32 L = n_lvl; L-- > 0;) {
        const u32 l0 = lvl[L], l1 = lvl[L + 1];
        for (u32 i = l0 + (u32)lane; i < l1; i += 32) {
            u32 a = order[i];
            u32 sib = t.tn_sib[base + a];
            u32 own = tree_open_len(sib) + tree_close_len(dpeer, P, a, parent[a], sib, plen_tmp[a]);
            u32 n = cnt[a], b0 = off[a], acc = 0;
            for (u32 k = 0; k < n; k++) { u32 c = child[b0 + k]; rel[c] = acc; acc += sub[c]; }
            sub[a] = own + acc;
            slot_tmp[a] = acc;   // bytes of the children: the distance between the node's two pieces
        }
        __syncwarp();
    }
    for (u32 c = lane; c < C; c += 32) {
        u32 n = cnt[A + c], b0 = off[A + c], acc = 0;
        for (u32 k = 0; k < n; k++) { u32 x = child[b0 + k]; rel[x] = acc; acc += sub[x]; }
        sub[A + c] = acc;
    }
    __syncwarp();
    // top-down: absolute offsets (1 = the container's '[')
    for (u32 L = 0; L < n_lvl; L++) {
        const u32 l0 = lvl[L], l1 = lvl[L + 1];
        for (u32 i = l0 + (u32)lane; i < l1; i += 32) {
            u32 a = order[i];
            u32 p = parent[a];
            u32 o = p == TREE_ROOT ? 1u + rel[a] : t.tn_aopen[base + p] + tree_open_len(t.tn_sib[base + p]) + rel[a];
            t.tn_aopen[base + a] = o;
            t.tn_aclose[base + a] = o + tree_open_len(t.tn_sib[base + a]) + slot_tmp[a];
        }
        __syncwarp();
    }
    if (lane == 0) docs[d].has_tree = has_meta ? 1u : 3u;   // bit1: the lane-parallel JSON layout is valid
}
