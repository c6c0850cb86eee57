// loro_b200 -- checkout: the state of a document at an earlier version.
//
// Replaces (reference, relative to crates/loro-internal/src):
//   loro.rs:1353-1433 LoroDoc::checkout(&frontiers) followed by get_deep_value (state at Frontiers F)
// The state at F is built from every atom in the causal closure of F and from nothing else.  Its version vector is
//   V = max over ids (p, c) of F of (vv of the change holding (p, c)) with V[p] >= c + 1,
// which this kernel writes as ck_end[peer slot].  k_op_classify then cuts every op row at V (a change that straddles V is
// cut inside, its op under the cut inside the op) and k_seq_integrate leaves its trackers at V; map LWW, the tree apply
// and the JSON only ever see what survived the cut.  An id of F that is not an applied atom of the document -- an unknown
// peer, a counter at or past the oplog vv, an id inside a pending change -- fails the document with DOC_ERR_FRONTIERS
// (LoroError::FrontiersNotFound, loro.rs:1394-1410).
#pragma once
#include "k_resolve.cuh"

#define CK_LATEST 0xFFFFFFFFu   // ck_range[d].x of a document without a request: it stays at the latest version

// warp per document, after k_doc_frontiers (it needs the applied copies and ch_vv of the causal scan).  The request of
// document d is the ids [ck_range[d].x, ck_range[d].y) of ck_peer / ck_ctr; an empty range is the empty version.
__global__ void k_doc_checkout(DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t,
                               const uint2* __restrict__ ck_range, const u64* __restrict__ ck_peer,
                               const i32* __restrict__ ck_ctr) {
    const u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    DocInfo& di = docs[d];
    if (di.code != DOC_OK) return;
    const u32 P = di.P;
    const DocPeer* dp = t.dpeer + di.peer0;
    i32* V = t.ck_end + di.peer0;   // lane l owns the peers q = l (mod 32): no two lanes write one entry
    const uint2 r = ck_range[d];
    if (r.x == CK_LATEST) {
        for (u32 q = lane; q < P; q += 32) V[q] = dp[q].end_counter;
        return;
    }
    for (u32 q = lane; q < P; q += 32) V[q] = 0;
    bool found = true;
    for (u32 f = r.x; f < r.y && found; f++) {
        const u64 pid = ck_peer[f];
        const i32 c = ck_ctr[f];
        u32 p = 0xFFFFFFFFu;
        for (u32 q0 = 0; q0 < P; q0 += 32) {
            unsigned m = __ballot_sync(LB_FULL, q0 + lane < P && dp[q0 + lane].id == pid);
            if (m) { p = q0 + (u32)(__ffs(m) - 1); break; }
        }
        // (p, c) must lie in an applied copy of p: their applied ranges ascend, lamport_of bisects them
        u32 lam, ch;
        found = p != 0xFFFFFFFFu && lamport_of(di, t, p, c, &lam, &ch);
        if (!found) break;
        const i32* row = t.ch_vv + di.vv0 + (u64)t.ch_pos[ch] * P;
        for (u32 q = lane; q < P; q += 32) {
            i32 v = row[q];
            if (q == p && c + 1 > v) v = c + 1;
            if (v > V[q]) V[q] = v;
        }
    }
    if (!found && lane == 0) di.code = LB_ERR(DOC_ERR_FRONTIERS);
}
