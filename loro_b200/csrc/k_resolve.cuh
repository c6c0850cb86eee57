// loro_b200 -- phase 3: per-document resolution and causal scan.
//
// Replaces (reference, relative to crates/loro-internal/src):
//   arena.rs register_container / keys / peers interning (doc-level tables)
//   encoding/outdated_encode_reordered.rs:40-83 import_changes_to_oplog (dedupe, lamport from deps, pending)
//   oplog/loro_dag.rs:935-954 get_lamport / get_change_lamport_from_deps
//   oplog/pending_changes.rs:31-140 (changes whose deps are missing stay pending)
//   oplog.rs:402-470 + dag/iter.rs:180-339 (a causal iteration order; the engine always replays from the
//   empty version, and prefers to stay on one peer's chain so that the tracker rarely has to retreat)
//   diff_calc.rs:175-236 (the version vector handed to each calculator before a change)
// Round-1 shape: one thread per document (documents are independent; a batch has 10^3..10^5 of them).
#pragma once
#include "lb_tables.cuh"

#define EPOCH_FP 0x80000000u
#define EPOCH_NEVER 0x7FFFFFFFu

__device__ inline bool bytes_eq(const u8* a, const u8* b, u32 n) {
    for (u32 i = 0; i < n; i++)
        if (a[i] != b[i]) return false;
    return true;
}

// thread per doc: intern peers / containers / keys, order the changes per peer.
__global__ void k_doc_tables(const u8* __restrict__ bytes, DocInfo* __restrict__ docs, u32 n_docs,
                             const BlockInfo* __restrict__ blocks, const __grid_constant__ BatchTables t) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    DocInfo di = docs[d];
    di.P = di.C = di.K = 0;
    di.n_changes = 0;
    di.n_ops = 0;
    if (di.code != DOC_OK) { docs[d] = di; return; }
    for (u32 b = di.b0; b < di.b1; b++)
        if (blocks[b].err) { di.code = blocks[b].err; break; }
    if (di.code != DOC_OK || di.b0 == di.b1) { docs[d] = di; return; }
    const BlockInfo& first = blocks[di.b0];
    const BlockInfo& end = blocks[di.b1];  // sentinel / next doc's first block holds the scan totals
    di.peer0 = first.peer0;
    di.cid0 = first.cid0;
    di.key0 = first.key0;
    di.ch0 = first.ch0;
    di.op0 = first.op0;
    di.n_changes = (u32)(end.ch0 - first.ch0);
    di.n_ops = end.op0 - first.op0;
    di.n_deps = (u32)(end.dep0 - first.dep0);
    di.P_cap = (u32)(end.peer0 - first.peer0);
    di.C_cap = (u32)(end.cid0 - first.cid0);
    di.K_cap = (u32)(end.key0 - first.key0);
    // ---- peers
    u32 P = 0;
    for (u32 b = di.b0; b < di.b1; b++) {
        const BlockInfo& bi = blocks[b];
        for (u32 j = 0; j < bi.n_peers; j++) {
            u64 id = t.peer_id[bi.peer0 + j];
            u32 f = 0;
            while (f < P && t.dpeer[di.peer0 + f].id != id) f++;
            if (f == P) {
                DocPeer np;
                np.id = id;
                np.rank = 0;
                np.succ_lo = 0;
                np.has_succ = 0;
                np.end_counter = 0;
                np.n_app = 0;
                np.atom_base = 0;
                np.ch_first = 0;
                np.ch_count = 0;
                np.pend_lo = 0;
                np.pend_hi = 0;
                t.dpeer[di.peer0 + P] = np;
                P++;
            }
            t.peer_map[bi.peer0 + j] = f;
        }
    }
    if (P > 0xFFF0) { di.code = LB_ERR(DOC_ERR_CAPACITY); docs[d] = di; return; }
    for (u32 i = 0; i < P; i++) {
        u32 r = 0;
        u64 id = t.dpeer[di.peer0 + i].id;
        for (u32 j = 0; j < P; j++) r += t.dpeer[di.peer0 + j].id < id;
        t.dpeer[di.peer0 + i].rank = r;
    }
    // ---- keys (dedupe by bytes)
    u32 K = 0;
    for (u32 b = di.b0; b < di.b1; b++) {
        const BlockInfo& bi = blocks[b];
        for (u32 j = 0; j < bi.n_keys; j++) {
            u64 off = t.key_off[bi.key0 + j];
            u32 len = t.key_len[bi.key0 + j];
            u32 f = 0;
            while (f < K && !(t.dkey_len[di.key0 + f] == len && bytes_eq(bytes + t.dkey_off[di.key0 + f], bytes + off, len))) f++;
            if (f == K) {
                t.dkey_off[di.key0 + K] = off;
                t.dkey_len[di.key0 + K] = len;
                K++;
            }
            t.key_map[bi.key0 + j] = f;
        }
    }
    // ---- containers
    u32 C = 0;
    for (u32 b = di.b0; b < di.b1; b++) {
        const BlockInfo& bi = blocks[b];
        for (u32 j = 0; j < bi.n_cids; j++) {
            u8 is_root = t.cid_root[bi.cid0 + j], type = t.cid_type[bi.cid0 + j];
            i32 koc = t.cid_koc[bi.cid0 + j];
            u64 peer = 0, noff = 0;
            u32 nlen = 0;
            if (is_root) {
                noff = t.key_off[bi.key0 + (u32)koc];
                nlen = t.key_len[bi.key0 + (u32)koc];
            } else
                peer = t.peer_id[bi.peer0 + t.cid_peer_idx[bi.cid0 + j]];
            u32 f = 0;
            for (; f < C; f++) {
                const DocContainer& dc = t.dcont[di.cid0 + f];
                if (dc.is_root != is_root || dc.type != type) continue;
                if (is_root) {
                    if (dc.name_len == nlen && bytes_eq(bytes + dc.name_off, bytes + noff, nlen)) break;
                } else if (dc.peer == peer && dc.counter == koc)
                    break;
            }
            if (f == C) {
                DocContainer dc;
                memset(&dc, 0, sizeof(dc));
                dc.is_root = is_root;
                dc.type = type;
                dc.name_off = noff;
                dc.name_len = nlen;
                dc.peer = peer;
                dc.counter = is_root ? 0 : koc;
                dc.key_or_peer = is_root ? t.key_map[bi.key0 + (u32)koc] : t.peer_map[bi.peer0 + t.cid_peer_idx[bi.cid0 + j]];
                t.dcont[di.cid0 + C] = dc;
                C++;
            }
            t.cid_map[bi.cid0 + j] = f;
        }
    }
    di.P = P;
    di.C = C;
    di.K = K;
    // ---- order blocks by (peer, counter_start) : insertion sort on the doc's slice of blk_order
    u32 nb = di.b1 - di.b0;
    for (u32 i = 0; i < nb; i++) {
        u32 b = di.b0 + i;
        u32 bp = t.peer_map[blocks[b].peer0];
        u32 bc = blocks[b].counter_start;
        u32 j = i;
        while (j > 0) {
            u32 o = t.blk_order[di.b0 + j - 1];
            u32 op = t.peer_map[blocks[o].peer0];
            if (op < bp || (op == bp && blocks[o].counter_start <= bc)) break;
            t.blk_order[di.b0 + j] = o;
            j--;
        }
        t.blk_order[di.b0 + j] = b;
    }
    // ---- per-peer change lists
    u32 k = 0;
    u32 cur_peer = 0xFFFFFFFFu;
    for (u32 i = 0; i < nb; i++) {
        const BlockInfo& bi = blocks[t.blk_order[di.b0 + i]];
        u32 p = t.peer_map[bi.peer0];
        if (p != cur_peer) {
            t.dpeer[di.peer0 + p].ch_first = k;
            cur_peer = p;
        }
        for (u32 c = 0; c < bi.n_changes; c++) {
            u32 ch = (u32)(bi.ch0 + c);
            t.ch_order[di.ch0 + k] = ch;
            t.ch_peer[ch] = (u16)p;
            k++;
        }
        t.dpeer[di.peer0 + p].ch_count += bi.n_changes;
    }
    // blocks of one blob never overlap, blocks of several blobs (import_batch) may: keep every peer's list ordered
    // by counter (stable, so a re-delivered change follows the first copy)
    for (u32 p = 0; p < P; p++) {
        const DocPeer& dp = t.dpeer[di.peer0 + p];
        u32* lst = t.ch_order + di.ch0 + dp.ch_first;
        for (u32 i = 1; i < dp.ch_count; i++) {
            u32 c = lst[i];
            i32 cc = t.ch_counter[c];
            u32 j = i;
            while (j > 0 && t.ch_counter[lst[j - 1]] > cc) { lst[j] = lst[j - 1]; j--; }
            lst[j] = c;
        }
    }
    docs[d] = di;
}

// lamport of atom (peer p, counter c) if applied; returns false when unknown.  The applied copies of a peer are kept in
// application order (ch_aorder): their applied ranges ascend, so the one holding c is found by bisection on the start.
__device__ inline bool lamport_of(const DocInfo& di, const BatchTables& t, u32 p, i32 c, u32* out,
                                  u32* ch_out) {
    const DocPeer& dp = t.dpeer[di.peer0 + p];
    if (c < 0 || c >= dp.end_counter || dp.n_app == 0) return false;
    const u32* lst = t.ch_aorder + di.ch0 + dp.ch_first;
    u32 lo = 0, hi = dp.n_app;
    while (hi - lo > 1) {
        u32 mid = (lo + hi) >> 1;
        if (t.ch_counter[lst[mid]] + (i32)t.ch_trim[lst[mid]] <= c) lo = mid;
        else hi = mid;
    }
    u32 ch = lst[lo];
    if (c < t.ch_counter[ch] + (i32)t.ch_trim[ch] || c >= t.ch_counter[ch] + (i32)t.ch_len[ch]) return false;
    *out = t.ch_lamport[ch] + (u32)(c - t.ch_counter[ch]);
    *ch_out = ch;
    return true;
}

// ---- import status of multi-blob documents.  T(copy) = max(rank of its blob, epoch of every atom it depends on);
// epoch(atom) = min T over the copies that cover it (whichever copy the reference meets first applies the atom, later
// ones are skipped or trimmed: oplog.rs:181-196); first-pass flag likewise.  Copies are visited in the order of the
// lamport of their first atom (a merge of the per-peer lists), so every copy covering a dependency has its T by then.
#define EPOCH_SCAN_CAP 512   // covering copies looked at per atom: a document with more copies stacked on one atom gets an
                             // approximate status (never a wrong state)
__device__ inline u32 atom_epoch(const DocInfo& di, const BatchTables& t, u32 p, i32 c) {
    const DocPeer& dp = t.dpeer[di.peer0 + p];
    if (c < 0 || c >= dp.end_counter) return EPOCH_NEVER;
    const u32* lst = t.ch_order + di.ch0 + dp.ch_first;
    const i32* mx = t.ch_maxend + di.ch0 + dp.ch_first;
    u32 lo = 0, hi = dp.ch_count;
    while (hi - lo > 1) {
        u32 mid = (lo + hi) >> 1;
        if (t.ch_counter[lst[mid]] <= c) lo = mid; else hi = mid;
    }
    u32 best = EPOCH_NEVER;
    for (u32 n = 0; n < EPOCH_SCAN_CAP; n++) {
        if (mx[lo] <= c) break;                      // nothing at or before `lo` reaches c
        u32 x = lst[lo];
        if (c < t.ch_counter[x] + (i32)t.ch_len[x]) {
            u32 e = t.ch_epoch[x];
            if ((e & ~EPOCH_FP) < (best & ~EPOCH_FP)) best = e;
            else if ((e & ~EPOCH_FP) == (best & ~EPOCH_FP)) best |= e & EPOCH_FP;
        }
        if (lo == 0) break;
        lo--;
    }
    return best;
}
__device__ inline u32 copy_epoch(const DocInfo& di, const BatchTables& t, const BlockInfo* blocks, u32 ch, u32 p) {
    const BlockInfo& bi = blocks[t.ch_block[ch]];
    const u32 k = bi.blob_rank;
    u32 E = k;
    bool fp = true;
    const u32 nd = t.ch_ndeps[ch] + (t.ch_dep_self[ch] ? 1u : 0u);
    for (u32 j = 0; j < nd; j++) {
        u32 dpi;
        i32 dc;
        if (j == t.ch_ndeps[ch]) { dpi = p; dc = t.ch_counter[ch] - 1; }
        else { dpi = t.peer_map[bi.peer0 + t.dep_peer_idx[t.ch_dep0[ch] + j]]; dc = t.dep_counter[t.ch_dep0[ch] + j]; }
        u32 ed = atom_epoch(di, t, dpi, dc);
        u32 e = ed & ~EPOCH_FP;
        if (e >= EPOCH_NEVER) return EPOCH_NEVER;
        if (e > E) E = e;
        if (e > k || (e == k && !(ed & EPOCH_FP))) fp = false;
    }
    return E | (fp ? EPOCH_FP : 0u);
}

// ---- multi-blob documents: WHICH copy of a change supplies an atom.  The reference imports a document's blobs one after
// the other, so an atom comes from the copy that can be applied first -- the lowest T = max(rank of its blob, epoch of
// its dependencies), a blob's first pass before its release of parked changes -- and later copies are skipped or trimmed
// (oplog.rs:181-196).  State does not care, exported bytes do: where a payload sits in the document's arenas, hence
// which neighbouring ops re-merge, depends on the blob that brought it.  Among the copies of peer p that can extend its
// frontier (consecutive in the counter-ordered list) the one with the lowest (T, parked, rank) is returned; *soft is set
// when some candidate's dependencies are not applied YET, i.e. a better copy may still turn up.  During the walk
// ch_epoch holds the epoch of every APPLIED copy (exact, because the copy applied for an atom is the reference's).
__device__ inline u32 pick_copy_multi(const DocInfo& di, const BatchTables& t, const BlockInfo* blocks, u32 p, u32 from,
                                      u32* lam_out, u32* epoch_out, bool* soft) {
    const DocPeer& dp = t.dpeer[di.peer0 + p];
    u32 best = 0xFFFFFFFFu, best_lam = 0, best_e = 0;
    u64 best_key = ~0ull;
    *soft = false;
    u32 looked = 0;
    for (u32 j = from; j < dp.ch_count; j++) {
        u32 ch = t.ch_order[di.ch0 + dp.ch_first + j];
        i32 ctr = t.ch_counter[ch];
        if (ctr > dp.end_counter) break;                                   // sorted by counter: nothing further reaches the frontier
        if (++looked > EPOCH_SCAN_CAP) break;   // hundreds of copies stacked on one atom: the first ones decide (a bound on
                                                // the work a hostile document can ask for; see EPOCH_SCAN_CAP)
        if (t.ch_applied[ch] || ctr + (i32)t.ch_len[ch] <= dp.end_counter) continue;   // consumed / already known
        const BlockInfo& bi = blocks[t.ch_block[ch]];
        const u32 k = bi.blob_rank;
        u32 E = k, lam = 0;
        bool fp = true, ready = true;
        const u32 nd = t.ch_ndeps[ch] + (t.ch_dep_self[ch] ? 1u : 0u);
        for (u32 q = 0; q < nd; q++) {
            u32 dpi;
            i32 dc;
            if (q == t.ch_ndeps[ch]) { dpi = p; dc = ctr - 1; }
            else { dpi = t.peer_map[bi.peer0 + t.dep_peer_idx[t.ch_dep0[ch] + q]]; dc = t.dep_counter[t.ch_dep0[ch] + q]; }
            u32 l, dch;
            if (!lamport_of(di, t, dpi, dc, &l, &dch)) { ready = false; break; }
            if (l + 1 > lam) lam = l + 1;
            u32 ed = t.ch_epoch[dch], e = ed & ~EPOCH_FP;
            if (e > E) E = e;
            if (e > k || (e == k && !(ed & EPOCH_FP))) fp = false;
        }
        if (!ready) { *soft = true; continue; }
        if (ctr < dp.end_counter) {          // applied as a slice: it follows its own predecessor (change.rs:248-252)
            u32 l, dch;
            if (!lamport_of(di, t, p, dp.end_counter - 1, &l, &dch)) { *soft = true; continue; }
            lam = l + 1;
        }
        u64 key = ((u64)E << 33) | ((u64)(fp ? 0u : 1u) << 32) | k;
        if (key < best_key) { best_key = key; best = j; best_lam = lam; best_e = E | (fp ? EPOCH_FP : 0u); }
    }
    *lam_out = best_lam;
    *epoch_out = best_e;
    return best;
}

__global__ void k_doc_causal(DocInfo* __restrict__ docs, u32 n_docs, const BlockInfo* __restrict__ blocks,
                             const __grid_constant__ BatchTables t, u32* __restrict__ peer_cursor, const u32* __restrict__ doc_blob0,
                             i32* __restrict__ pend_scratch) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    DocInfo di = docs[d];
    di.n_applied = 0;
    di.n_pending = 0;
    di.atom_ops = 0;
    di.atom_total = 0;
    if (di.code != DOC_OK || di.n_changes == 0) { docs[d] = di; return; }
    u32 P = di.P;
    u32* cursor = peer_cursor + di.peer0;  // per peer: index of the next unapplied change
    for (u32 p = 0; p < P; p++) cursor[p] = 0;
    u32 cur = 0xFFFFFFFFu;
    u32 walk_n = 0;
    const bool multi_blob = di.n_blobs > 1 && t.ch_epoch != nullptr;
    while (true) {
        // ---- pick a ready change: stay on the current peer if possible, else min (lamport, peer)
        u32 pick = 0xFFFFFFFFu, pick_lam = 0, pick_ch = 0, pick_e = EPOCH_FP;
        u32 soft_pick = 0xFFFFFFFFu, soft_lam = 0, soft_ch = 0, soft_e = 0;
        for (u32 step = 0; step < P + 1; step++) {
            u32 p;
            if (step == 0) { if (cur == 0xFFFFFFFFu) continue; p = cur; }
            else { p = step - 1; if (p == cur) continue; }
            DocPeer& dp = t.dpeer[di.peer0 + p];
            if (cursor[p] >= dp.ch_count) continue;
            if (multi_blob) {
                // consumed and known copies at the front are done with
                while (cursor[p] < dp.ch_count) {
                    u32 c0 = t.ch_order[di.ch0 + dp.ch_first + cursor[p]];
                    if (t.ch_applied[c0] || t.ch_counter[c0] + (i32)t.ch_len[c0] <= dp.end_counter) cursor[p]++; else break;
                }
                if (cursor[p] >= dp.ch_count) continue;
                u32 lam_m, e_m;
                bool soft;
                u32 j = pick_copy_multi(di, t, blocks, p, cursor[p], &lam_m, &e_m, &soft);
                if (j == 0xFFFFFFFFu) continue;
                u32 chm = t.ch_order[di.ch0 + dp.ch_first + j];
                if (soft) {      // a better copy may still become ready: only taken when nothing else can move
                    if (soft_pick == 0xFFFFFFFFu) { soft_pick = p; soft_lam = lam_m; soft_ch = chm; soft_e = e_m; }
                    continue;
                }
                if (step == 0) { pick = p; pick_lam = lam_m; pick_ch = chm; pick_e = e_m; break; }
                if (pick == 0xFFFFFFFFu || lam_m < pick_lam ||
                    (lam_m == pick_lam && t.dpeer[di.peer0 + p].rank < t.dpeer[di.peer0 + pick].rank)) {
                    pick = p; pick_lam = lam_m; pick_ch = chm; pick_e = e_m;
                }
                continue;
            }
            u32 ch = t.ch_order[di.ch0 + dp.ch_first + cursor[p]];
            i32 ctr = t.ch_counter[ch];
            if (ctr != dp.end_counter) {
                if (ctr < dp.end_counter) {  // overlapping duplicate: drop if fully covered
                    if (ctr + (i32)t.ch_len[ch] <= dp.end_counter) { cursor[p]++; step--; continue; }
                    // partial overlap (an update exported from an older version vector): the known part is trimmed and
                    // the rest applies as Change::slice -- it depends on its own predecessor only (change.rs:248-252)
                    u32 l, c2;
                    if (!lamport_of(di, t, p, dp.end_counter - 1, &l, &c2)) continue;
                    u32 lam_t = l + 1;
                    if (step == 0) { pick = p; pick_lam = lam_t; pick_ch = ch; break; }
                    if (pick == 0xFFFFFFFFu || lam_t < pick_lam ||
                        (lam_t == pick_lam && t.dpeer[di.peer0 + p].rank < t.dpeer[di.peer0 + pick].rank)) {
                        pick = p; pick_lam = lam_t; pick_ch = ch;
                    }
                }
                continue;  // gap: predecessor missing -> pending
            }
            bool ok = true;
            u32 lam = 0;
            if (t.ch_dep_self[ch]) {
                u32 l, c2;
                if (!lamport_of(di, t, p, ctr - 1, &l, &c2)) ok = false; else lam = l + 1;
            }
            u64 d0 = t.ch_dep0[ch];
            u32 bpeer0 = (u32)0;
            const BlockInfo& bi = blocks[t.ch_block[ch]];
            (void)bpeer0;
            for (u32 k = 0; ok && k < t.ch_ndeps[ch]; k++) {
                u32 dp_idx = t.peer_map[bi.peer0 + t.dep_peer_idx[d0 + k]];
                u32 l, c2;
                if (!lamport_of(di, t, dp_idx, t.dep_counter[d0 + k], &l, &c2)) ok = false;
                else if (l + 1 > lam) lam = l + 1;
            }
            if (!ok) continue;
            if (step == 0) { pick = p; pick_lam = lam; pick_ch = ch; break; }
            if (pick == 0xFFFFFFFFu || lam < pick_lam ||
                (lam == pick_lam && t.dpeer[di.peer0 + p].rank < t.dpeer[di.peer0 + pick].rank)) {
                pick = p; pick_lam = lam; pick_ch = ch;
            }
        }
        if (pick == 0xFFFFFFFFu && soft_pick != 0xFFFFFFFFu) { pick = soft_pick; pick_lam = soft_lam; pick_ch = soft_ch; pick_e = soft_e; }
        if (pick == 0xFFFFFFFFu || di.code != DOC_OK) break;
        // ---- apply
        u32 ch = pick_ch;
        DocPeer& dp = t.dpeer[di.peer0 + pick];
        i32 ctr = t.ch_counter[ch];
        const u32 trim = ctr < dp.end_counter ? (u32)(dp.end_counter - ctr) : 0u;
        u32 local = dp.ch_first + dp.n_app;  // its place in the peer's applied order = row of this change in the doc's ch_vv
        i32* v = t.ch_vv + di.vv0 + (u64)local * P;
        for (u32 q = 0; q < P; q++) v[q] = 0;
        const BlockInfo& bi = blocks[t.ch_block[ch]];
        u32 ndeps = trim ? 1u : t.ch_ndeps[ch] + (t.ch_dep_self[ch] ? 1 : 0);
        for (u32 k = 0; k < ndeps; k++) {
            u32 dpi;
            i32 dc;
            if (trim) { dpi = pick; dc = dp.end_counter - 1; }
            else if (k == t.ch_ndeps[ch]) { dpi = pick; dc = ctr - 1; }
            else { dpi = t.peer_map[bi.peer0 + t.dep_peer_idx[t.ch_dep0[ch] + k]]; dc = t.dep_counter[t.ch_dep0[ch] + k]; }
            u32 l = 0, dch = ch;
            lamport_of(di, t, dpi, dc, &l, &dch);
            const i32* dv = t.ch_vv + di.vv0 + (u64)t.ch_pos[dch] * P;   // the dependency is applied: its row is known
            for (u32 q = 0; q < P; q++) if (dv[q] > v[q]) v[q] = dv[q];
            if (dc + 1 > v[dpi]) v[dpi] = dc + 1;
        }
        t.ch_lamport[ch] = pick_lam - trim;   // lamport of the change's (trimmed) first atom: counters and lamports run in step
        t.ch_trim[ch] = trim;
        if (multi_blob) t.ch_epoch[ch] = pick_e;
        t.ch_applied[ch] = 1;
        t.ch_pos[ch] = local;
        t.ch_aorder[di.ch0 + local] = ch;
        dp.n_app++;
        t.ch_walk[di.ch0 + walk_n++] = ch;
        dp.end_counter = ctr + (i32)t.ch_len[ch];
        di.atom_ops += t.ch_len[ch] - trim;
        if (!multi_blob) cursor[pick]++;     // (multi-blob: the cursor skips consumed copies when the peer is looked at again)
        cur = pick;
    }
    di.n_applied = walk_n;
    // the copies that were not applied (dropped duplicates, pending changes) follow the applied ones
    for (u32 p = 0; p < P; p++) {
        const DocPeer& dp = t.dpeer[di.peer0 + p];
        u32 w = dp.n_app;
        for (u32 k = 0; k < dp.ch_count; k++) {
            u32 ch = t.ch_order[di.ch0 + dp.ch_first + k];
            if (!t.ch_applied[ch]) t.ch_aorder[di.ch0 + dp.ch_first + w++] = ch;
        }
    }
    // ---- import status + atom bases.  ImportStatus of LoroDoc::import_batch (loro.rs:1183-1290) folds the statuses of
    // the blobs imported one after the other: success[peer] = (start of the first blob that applied something of the
    // peer, highest end) -- atoms of a peer apply in counter order, so that is [first counter a new blob applied, end);
    // pending[peer] = (min start, MIN end) over the blobs of the hull of the changes each blob parked in its first pass
    // (encoding.rs:252-257), whether or not a later step released them.  Blobs below n_prior restate the earlier state
    // of the document (lb_docset_import) and report nothing.
    const bool multi = di.n_blobs > 1 && t.ch_maxend && pend_scratch;
    if (multi) {
        // T of every copy, in the order of the lamport of its first atom
        for (u32 p = 0; p < P; p++) {
            const DocPeer& dp = t.dpeer[di.peer0 + p];
            i32 m = -1;
            for (u32 k = 0; k < dp.ch_count; k++) {
                u32 ch = t.ch_order[di.ch0 + dp.ch_first + k];
                i32 e = t.ch_counter[ch] + (i32)t.ch_len[ch];
                if (e > m) m = e;
                t.ch_maxend[di.ch0 + dp.ch_first + k] = m;
                t.ch_epoch[ch] = EPOCH_NEVER;
            }
            cursor[p] = 0;
            t.head_lamport[di.peer0 + p] = 0xFFFFFFFFu;
            if (dp.ch_count) {
                u32 l, c2;
                if (lamport_of(di, t, p, t.ch_counter[t.ch_order[di.ch0 + dp.ch_first]], &l, &c2)) t.head_lamport[di.peer0 + p] = l;
            }
        }
        while (true) {
            u32 bp = 0xFFFFFFFFu, bl = 0xFFFFFFFFu;
            for (u32 p = 0; p < P; p++) {
                u32 l = t.head_lamport[di.peer0 + p];
                if (l < bl) { bl = l; bp = p; }
            }
            if (bp == 0xFFFFFFFFu) break;      // what is left starts beyond the document's version: never applied
            const DocPeer& dp = t.dpeer[di.peer0 + bp];
            u32 ch = t.ch_order[di.ch0 + dp.ch_first + cursor[bp]];
            t.ch_epoch[ch] = copy_epoch(di, t, blocks, ch, bp);
            cursor[bp]++;
            u32 nl = 0xFFFFFFFFu;
            if (cursor[bp] < dp.ch_count) {
                u32 l, c2;
                if (lamport_of(di, t, bp, t.ch_counter[t.ch_order[di.ch0 + dp.ch_first + cursor[bp]]], &l, &c2)) nl = l;
            }
            t.head_lamport[di.peer0 + bp] = nl;
        }
    }
    u32 base = 0;
    const u32 nb_new = di.n_blobs - di.n_prior;
    i32* hull = (multi && nb_new > 1) ? pend_scratch + 2 * (u64)(doc_blob0[d] + di.n_prior) : nullptr;
    for (u32 p = 0; p < P; p++) {
        DocPeer& dp = t.dpeer[di.peer0 + p];
        dp.atom_base = base;
        base += (u32)dp.end_counter;
        dp.pend_lo = dp.pend_hi = 0;
        dp.has_succ = 0;
        dp.succ_lo = 0;
        if (hull) for (u32 k = 0; k < nb_new; k++) { hull[2 * k] = 0x7FFFFFFF; hull[2 * k + 1] = -1; }
        i32 prior_end = -1;     // the atoms below it were in the document before this import
        for (u32 k = 0; k < dp.ch_count; k++) {
            u32 ch = t.ch_order[di.ch0 + dp.ch_first + k];
            i32 c0 = t.ch_counter[ch], c1 = c0 + (i32)t.ch_len[ch];
            const u32 rank = blocks[t.ch_block[ch]].blob_rank;
            bool parked;
            if (!multi) {
                // one blob: what it cannot apply stays parked, everything else applies in its first pass
                if (t.ch_applied[ch]) { if (prior_end < 0) prior_end = c0 + (i32)t.ch_trim[ch]; continue; }
                if (c1 <= dp.end_counter) continue;
                parked = true;
                di.n_pending++;
            } else {
                u32 e = t.ch_epoch[ch];
                if ((e & ~EPOCH_FP) < di.n_prior) { if (c1 > prior_end) prior_end = c1; }
                else if (prior_end < 0 && t.ch_applied[ch] && di.n_prior == 0) prior_end = c0 + (i32)t.ch_trim[ch];
                if (!t.ch_applied[ch] && c1 > dp.end_counter) di.n_pending++;
                if ((e & ~EPOCH_FP) >= EPOCH_NEVER) parked = true;
                else {
                    // known when its own blob arrived (all of it applied by an earlier blob)?  then it was skipped
                    if ((atom_epoch(di, t, p, c1 - 1) & ~EPOCH_FP) < rank) continue;
                    parked = !(e & EPOCH_FP);
                }
            }
            if (!parked || rank < di.n_prior) continue;
            if (hull) {
                i32* h = hull + 2 * (rank - di.n_prior);
                if (c0 < h[0]) h[0] = c0;
                if (c1 > h[1]) h[1] = c1;
            } else if (dp.pend_lo == dp.pend_hi) { dp.pend_lo = c0; dp.pend_hi = c1; }
            else { if (c0 < dp.pend_lo) dp.pend_lo = c0; if (c1 > dp.pend_hi) dp.pend_hi = c1; }
        }
        if (prior_end < 0) prior_end = 0;
        if (dp.end_counter > prior_end) { dp.has_succ = 1; dp.succ_lo = prior_end; }
        if (hull) {
            bool any = false;
            for (u32 k = 0; k < nb_new; k++) {
                if (hull[2 * k + 1] < 0) continue;
                if (!any) { dp.pend_lo = hull[2 * k]; dp.pend_hi = hull[2 * k + 1]; any = true; }
                else { if (hull[2 * k] < dp.pend_lo) dp.pend_lo = hull[2 * k]; if (hull[2 * k + 1] < dp.pend_hi) dp.pend_hi = hull[2 * k + 1]; }
            }
        }
    }
    di.atom_total = base;
    docs[d] = di;
}

// thread per doc: frontiers = the heads of the causal graph (reference: version/frontiers.rs:233-246
// update_frontiers_on_new_change, oplog/loro_dag.rs:251-269).  The last id of peer p is a head unless it lies in the
// causal past of another peer's change; version vectors grow along a peer's chain, so looking at every peer's LAST
// applied change is enough.
__global__ void k_doc_frontiers(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK) return;
    u32 P = di.P;
    for (u32 p = 0; p < P; p++) t.dpeer[di.peer0 + p].is_head = t.dpeer[di.peer0 + p].end_counter > 0 ? 1u : 0u;
    for (u32 q = 0; q < P; q++) {
        const DocPeer& dq = t.dpeer[di.peer0 + q];
        // last applied change of q
        if (dq.n_app == 0) continue;
        u32 last = t.ch_aorder[di.ch0 + dq.ch_first + dq.n_app - 1];
        const i32* v = t.ch_vv + di.vv0 + (u64)t.ch_pos[last] * P;
        for (u32 p = 0; p < P; p++)
            if (p != q && v[p] >= t.dpeer[di.peer0 + p].end_counter && t.dpeer[di.peer0 + p].end_counter > 0) t.dpeer[di.peer0 + p].is_head = 0;
    }
}
