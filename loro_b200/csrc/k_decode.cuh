// loro_b200 -- phase 2: change-block decode into batch-wide SoA tables.
//
// Replaces (reference, relative to crates/loro-internal/src):
//   oplog/change_store/block_encode.rs:95-119 (EncodedBlock envelope), :527-659 (decode_block)
//   oplog/change_store/block_meta_encode.rs:90-179 (decode_changes_header)
//   encoding/arena.rs:94-101 (ContainerArena), block_encode.rs:290-300 (keys)
//   encoding/value.rs:343-391, 603-700 (values stream), encoding/outdated_encode_reordered.rs:215-423
//   third-party serde_columnar 0.3.14 column codecs (docs/encoding.md:1056-1398)
// Round-1 shape: one thread per block, two passes (count -> host allocates -> fill).  Blocks are ~4 KB and a
// batch holds 10^5..10^6 of them, so the parallelism is across blocks.
#pragma once
#include "lb_tables.cuh"

// ---- skip one LoroValue (kind byte already consumed) ; iterative, bounded depth
// reference: value.rs:620-700 read_value_content
// scalar LoroValue kinds (everything but List / Map): skipped without the explicit stack
__device__ __forceinline__ bool skip_loro_scalar(Cur& c, u8 kind, u32* n_child_containers) {
    switch (kind) {
        case 0: case 1: case 2: return true;
        case 3: (void)c.sleb(); return true;
        case 4: c.skip(8); return true;
        case 5: case 6: { u64 n = c.varint(); c.skip(n); return true; }
        case 9: (void)c.get(); if (n_child_containers) (*n_child_containers)++; return true;
        default: return false;
    }
}
__device__ inline void skip_loro_value_content(Cur& c, u8 kind, u32* n_child_containers, u32* n_maps = nullptr) {
    // fast paths: a scalar, or a list of scalars (what a List insert carries) -- no stack, no local memory
    if (skip_loro_scalar(c, kind, n_child_containers)) return;
    if (kind == 7) {
        Cur save = c;
        u64 n = c.varint();
        bool flat = n <= (1u << 28);
        u32 kids = 0;
        for (u64 i = 0; flat && i < n && !c.err; i++) {
            u8 k = c.get();
            if (!skip_loro_scalar(c, k, &kids)) flat = false;
        }
        if (flat) { if (n_child_containers) *n_child_containers += kids; return; }
        c = save;          // nested content: start over on the general path
    }
    // stack of remaining item counts; bit 31 marks a map level (items carry a key index).  The decoder is the one walker
    // that meets values deeper than LB_MAX_NESTING: it rejects them, so every later walker's stack of that size fits.
    u32 stack[LB_MAX_NESTING];
    int sp = 0;
    bool have = true;  // a value of `kind` must be consumed now
    while (true) {
        if (have) {
            switch (kind) {
                case 0: case 1: case 2: break;
                case 3: (void)c.sleb(); break;
                case 4: c.skip(8); break;
                case 5: case 6: { u64 n = c.varint(); c.skip(n); break; }
                case 7: case 8: {
                    u64 n = c.varint();
                    if (n > (1u << 28)) { c.err = 1; return; }
                    if (sp >= LB_MAX_NESTING) { c.err = CUR_ERR_DEEP; return; }
                    stack[sp++] = (u32)n | (kind == 8 ? 0x80000000u : 0);
                    if (kind == 8 && n_maps) (*n_maps)++;
                    break;
                }
                case 9: (void)c.get(); if (n_child_containers) (*n_child_containers)++; break;
                default: c.err = 1; return;
            }
            have = false;
        }
        if (c.err) return;
        // pop finished levels
        while (sp > 0 && (stack[sp - 1] & 0x7fffffffu) == 0) sp--;
        if (sp == 0) return;
        stack[sp - 1]--;
        if (stack[sp - 1] & 0x80000000u) (void)c.varint();  // map key index
        kind = c.get();
        have = true;
    }
}

// length in bytes of the value of op kind `vt` starting at c (advances c)
__device__ inline void skip_value(Cur& c, u8 vt, u32* n_maps = nullptr) {
    switch (vt) {
        case VK_NULL: case VK_TRUE: case VK_FALSE: case VK_DELETE_ONCE: case VK_DELETE_SEQ: break;
        case VK_I64: case VK_DELTA_INT: (void)c.sleb(); break;
        case VK_F64: c.skip(8); break;
        case VK_STR: case VK_BINARY: { u64 n = c.varint(); c.skip(n); break; }
        case VK_CONTAINER: (void)c.varint(); break;
        case VK_LORO_VALUE: { u8 k = c.get(); skip_loro_value_content(c, k, nullptr, n_maps); break; }
        case VK_MARK_START: {
            (void)c.get(); (void)c.varint(); (void)c.varint();
            u8 k = c.get();
            skip_loro_value_content(c, k, nullptr);
            break;
        }
        case VK_TREE_MOVE: {
            (void)c.varint();
            u8 pn = c.get();
            (void)c.varint();
            if (!pn) (void)c.varint();
            break;
        }
        case VK_RAW_TREE_MOVE: {
            (void)c.varint(); (void)c.varint(); (void)c.varint();
            u8 pn = c.get();
            if (!pn) { (void)c.varint(); (void)c.varint(); }
            break;
        }
        case VK_LIST_MOVE: (void)c.varint(); (void)c.varint(); (void)c.varint(); break;
        case VK_LIST_SET: {
            (void)c.varint(); (void)c.varint();
            u8 k = c.get();
            skip_loro_value_content(c, k, nullptr);
            break;
        }
        default:
            if (vt & 0x80) { u64 n = c.varint(); c.skip(n); }  // Future kinds: binary payload
            else c.err = 1;
    }
}

// columnar wrapper: varint(1) varint(ncols) then per column varint(len)+payload
__device__ inline bool columnar_open(const u8* b, size_t n, int ncols, const u8** col, u32* col_len) {
    Cur c(b, n);
    if (c.varint() != 1) return false;
    if (c.varint() != (u64)ncols) return false;
    for (int i = 0; i < ncols; i++) {
        u64 len = c.varint();
        col[i] = c.p;
        col_len[i] = (u32)len;
        c.skip(len);
    }
    return !c.err && c.empty();
}

// ---------------------------------------------------------------- pass 1: envelope + counts
__global__ void k_block_count(const u8* __restrict__ bytes, BlockInfo* __restrict__ blocks, u64 n_blocks) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_blocks) return;
    BlockInfo bi = blocks[i];
    const u8* b = bytes + bi.off;
    Cur c(b, bi.len);
    bi.counter_start = (u32)c.varint();
    bi.counter_len = (u32)c.varint();
    bi.lamport_start = (u32)c.varint();
    bi.lamport_len = (u32)c.varint();
    bi.n_changes = (u32)c.varint();
    for (int s = 0; s < 8; s++) {
        u64 len = c.varint();
        bi.sec_off[s] = (u32)(c.p - b);
        bi.sec_len[s] = (u32)len;
        c.skip(len);
    }
    u32 err = 0;
    if (c.err || !c.empty() || bi.n_changes == 0 || bi.n_changes > bi.len) err = LB_ERR(DOC_ERR_DECODE);   // a change costs >= 1 byte
    bi.n_peers = bi.n_keys = bi.n_cids = bi.n_ops = bi.n_dels = bi.n_deps = 0;
    bi.n_pos = bi.pos_bytes = bi.n_tree = 0;
    bi.values_bytes = bi.sec_len[7];
    if (!err) {
        u32 N = bi.n_changes;
        // header: peers, N-1 lens, BoolRle(N), AnyRle dep_len(N) -> n_deps
        Cur h(b + bi.sec_off[0], bi.sec_len[0]);
        u64 np = h.varint();
        h.skip(8 * np);
        for (u32 k = 0; k + 1 < N && !h.err; k++) (void)h.varint();
        u64 got = 0;
        while (got < N && !h.err) { u64 run = h.varint(); if (run > N) { h.err = 1; break; } got += run; }  // BoolRle run lengths
        if (got != N) h.err = 1;
        got = 0;
        u64 ndeps = 0;
        while (got < N && !h.err) {  // AnyRle<usize>
            i64 sl = h.zigzag();
            if (sl == 0) { h.err = 1; break; }
            if (sl > 0) { u64 v = h.varint(); if (v > 0xFFFFFFFFull || (u64)sl > N) { h.err = 1; break; } ndeps += v * (u64)sl; got += (u64)sl; }
            else {
                if ((u64)(-sl) > N) { h.err = 1; break; }   // a literal run longer than the change count: corrupt
                for (i64 k = 0; k < -sl && !h.err; k++) ndeps += h.varint();
                got += (u64)(-sl);
            }
            if (ndeps > 0xFFFFFFFFull) { h.err = 1; break; }
        }
        if (got != N || np == 0 || np > 0xFFF0) h.err = 1;
        bi.n_peers = (u32)np;
        bi.n_deps = (u32)ndeps;
        // keys
        Cur k(b + bi.sec_off[3], bi.sec_len[3]);
        u32 nk = 0;
        while (!k.empty() && !k.err) { u64 len = k.varint(); k.skip(len); nk++; }
        bi.n_keys = nk;
        // cids
        Cur cc(b + bi.sec_off[2], bi.sec_len[2]);
        bi.n_cids = (u32)cc.varint();
        // ops: rows = sum |segment len| of the value_type column; dels = rows with kind DeleteSeq
        const u8* col[4];
        u32 col_len[4];
        bool ok = columnar_open(b + bi.sec_off[5], bi.sec_len[5], 4, col, col_len);
        u64 nops = 0, ndel = 0, ntree = 0;
        if (ok) {
            Cur v(col[2], col_len[2]);
            while (!v.empty() && !v.err) {
                i64 sl = v.zigzag();
                if (sl == 0 || sl > (i64)0x7FFFFFFF || sl < -(i64)0x7FFFFFFF) { v.err = 1; break; }
                if (sl > 0) { u8 x = v.get(); nops += (u64)sl; if (x == VK_DELETE_SEQ) ndel += (u64)sl; if (x == VK_RAW_TREE_MOVE) ntree += (u64)sl; }
                else {
                    for (i64 q = 0; q < -sl && !v.err; q++) { u8 x = v.get(); if (x == VK_DELETE_SEQ) ndel++; if (x == VK_RAW_TREE_MOVE) ntree++; }
                    nops += (u64)(-sl);
                }
                if (nops > 0x7FFFFFFFull) { v.err = 1; break; }
            }
            if (v.err) ok = false;
        }
        bi.n_ops = (u32)nops;
        bi.n_dels = (u32)ndel;
        bi.n_tree = (u32)ntree;
        // positions arena (arena.rs:159-233): column 0 = common prefix lengths (AnyRle<usize>), column 1 = the rests
        // (varint n, then n length-prefixed byte strings); sizes of the expanded positions are summed here
        if (ok && bi.sec_len[4]) {
            const u8* pc[2];
            u32 pl[2];
            if (!columnar_open(b + bi.sec_off[4], bi.sec_len[4], 2, pc, pl)) ok = false;
            else {
                RleCur pre(pc[0], pl[0], 1);
                Cur rest(pc[1], pl[1]);
                u64 np_ = rest.varint(), total = 0, last = 0;
                if (np_ > bi.sec_len[4]) ok = false;
                for (u64 q = 0; ok && q < np_; q++) {
                    i64 common;
                    if (!pre.next(&common)) { ok = false; break; }
                    u64 len = rest.varint();
                    rest.skip(len);
                    if (rest.err || common < 0 || (u64)common > last) { ok = false; break; }
                    last = (u64)common + len;
                    total += last;
                    if (total > 0x7FFFFFFFull) { ok = false; break; }
                }
                i64 extra;
                if (ok && (pre.next(&extra) || pre.c.err || !rest.empty())) ok = false;
                bi.n_pos = (u32)np_;
                bi.pos_bytes = (u32)total;
            }
        }
        if (h.err || k.err || cc.err || !ok || nops == 0) err = LB_ERR(DOC_ERR_DECODE);
        // run-length codes let a few bytes announce billions of rows: table sizes come from these counts, so a block
        // whose counts are out of proportion to its bytes is rejected here (one bad blob must not sink the batch).
        // Reference blocks stay below MAX_BLOCK_SIZE of estimated content, i.e. ~1.4 k rows.
        u64 cap = 8ull * bi.len + 64;
        if (nops > cap || ndeps > cap || N > cap || bi.n_cids > cap || bi.counter_len > (1u << 30) || nops > bi.counter_len)
            err = LB_ERR(DOC_ERR_DECODE);
        // an expanded position is at most the whole arena long: quadratic blow-ups (every entry re-using a long
        // prefix) are legal but bounded here so that one block cannot claim gigabytes
        if (bi.pos_bytes > 64u * bi.len + 4096u) err = LB_ERR(DOC_ERR_DECODE);
    }
    bi.err = err;
    if (err) { bi.n_peers = bi.n_keys = bi.n_cids = bi.n_ops = bi.n_dels = bi.n_deps = 0; bi.n_changes = 0; bi.n_pos = bi.pos_bytes = bi.n_tree = 0; }
    blocks[i] = bi;
}

enum { TRP_ROOT = 0, TRP_NODE = 1, TRP_DELETED = 2 };

// ---------------------------------------------------------------- pass 2: fill
// The block decoder in three single-thread pieces (`b` = the block's bytes, in global or in shared memory):
//   decode_block_small      header, change meta, keys, cids, positions   (tens of bytes per block)
//   decode_block_rows_cols  delete-start ids, the four ops columns, the values walk   (the bulk)
//   decode_block_fail       a failed block still leaves its rows pointing at its own changes
// k_block_decode_cols (the default) runs them one thread per block.  k_block_decode_warp (k_decode_warp.cuh) stages the
// block in shared memory and replaces decode_block_rows_cols by lane-parallel column expansion and value-chain
// resolution; the blocks its fast path does not cover still go through decode_block_rows_cols, on one lane.
__device__ inline u32 decode_block_small(const u8* b, const BlockInfo& bi, u64 i, const BatchTables& t) {
    u32 N = bi.n_changes;
    u32 err = 0;
    // ---- header
    Cur h(b + bi.sec_off[0], bi.sec_len[0]);
    u64 np = h.varint();
    for (u32 p = 0; p < bi.n_peers; p++) {
        u64 id = 0;
        for (int k = 0; k < 8; k++) id |= (u64)h.get() << (8 * k);
        t.peer_id[bi.peer0 + p] = id;
    }
    (void)np;
    // change lengths (N-1 explicit, last inferred)
    {
        i64 sum = 0;
        i32 ctr = (i32)bi.counter_start;
        for (u32 k = 0; k < N; k++) {
            i64 len;
            if (k + 1 < N) { len = (i64)h.varint(); sum += len; }
            else len = (i64)bi.counter_len - sum;
            if (len <= 0) err = LB_ERR(DOC_ERR_DECODE);
            t.ch_block[bi.ch0 + k] = (u32)i;
            t.ch_counter[bi.ch0 + k] = ctr;
            t.ch_len[bi.ch0 + k] = (u32)len;
            ctr += (i32)len;
        }
    }
    // dep_on_self BoolRle (N)
    {
        u32 got = 0;
        u8 state = 0;
        while (got < N && !h.err) {
            u64 run = h.varint();
            if (got + run > N) { h.err = 1; break; }
            for (u64 q = 0; q < run; q++) t.ch_dep_self[bi.ch0 + got + q] = state;
            got += (u32)run;
            state ^= 1;
        }
    }
    // dep_len AnyRle<usize> (N)
    {
        u32 got = 0;
        u64 dep = bi.dep0;
        while (got < N && !h.err) {
            i64 sl = h.zigzag();
            if (sl == 0) { h.err = 1; break; }
            u64 cnt = sl > 0 ? (u64)sl : (u64)(-sl);
            if (got + cnt > N) { h.err = 1; break; }
            u64 v = 0;
            if (sl > 0) v = h.varint();
            for (u64 q = 0; q < cnt; q++) {
                if (sl < 0) v = h.varint();
                t.ch_dep0[bi.ch0 + got + q] = dep;
                t.ch_ndeps[bi.ch0 + got + q] = (u32)v;
                dep += v;
            }
            got += (u32)cnt;
        }
        if (dep - bi.dep0 != bi.n_deps) h.err = 1;
    }
    // dep peer idx AnyRle<usize> (n_deps)
    {
        u32 got = 0;
        while (got < bi.n_deps && !h.err) {
            i64 sl = h.zigzag();
            if (sl == 0) { h.err = 1; break; }
            u64 cnt = sl > 0 ? (u64)sl : (u64)(-sl);
            if (got + cnt > bi.n_deps) { h.err = 1; break; }
            u64 v = 0;
            if (sl > 0) v = h.varint();
            for (u64 q = 0; q < cnt; q++) {
                if (sl < 0) v = h.varint();
                if (v >= bi.n_peers) err = LB_ERR(DOC_ERR_CORRUPT);
                t.dep_peer_idx[bi.dep0 + got + q] = (u32)v;
            }
            got += (u32)cnt;
        }
    }
    // dep counters DeltaOfDelta (n_deps)
    {
        DodCur d;
        d.begin(&h);
        if (bi.n_deps == 0 && d.has_first) h.err = 1;
        for (u32 k = 0; k < bi.n_deps; k++) t.dep_counter[bi.dep0 + k] = (i32)d.next(k == 0);
        d.finish();
    }
    // lamports DeltaOfDelta (N-1) ; last = lamport_start + lamport_len - last_len (block_meta_encode.rs:162)
    {
        DodCur d;
        d.begin(&h);
        for (u32 k = 0; k + 1 < N; k++) t.ch_lamport_wire[bi.ch0 + k] = (u32)d.next(k == 0);
        d.finish();
        t.ch_lamport_wire[bi.ch0 + N - 1] = bi.lamport_start + bi.lamport_len - t.ch_len[bi.ch0 + N - 1];
    }
    if (h.err || !h.empty()) err = err ? err : LB_ERR(DOC_ERR_DECODE);
    // ---- change meta: timestamps DoD (N), commit-message lengths AnyRle<u32> (N), message bytes
    {
        Cur m(b + bi.sec_off[1], bi.sec_len[1]);
        DodCur d;
        d.begin(&m);
        for (u32 k = 0; k < N; k++) t.ch_ts[bi.ch0 + k] = d.next(k == 0);
        d.finish();
        u32 got = 0;
        while (got < N && !m.err) {
            i64 sl = m.zigzag();
            if (sl == 0) { m.err = 1; break; }
            u64 cnt = sl > 0 ? (u64)sl : (u64)(-sl);
            if (got + cnt > N) { m.err = 1; break; }
            u64 v = 0;
            if (sl > 0) v = m.varint();
            for (u64 q = 0; q < cnt; q++) {
                if (sl < 0) v = m.varint();
                t.ch_msg_len[bi.ch0 + got + q] = (u32)v;
            }
            got += (u32)cnt;
        }
        u64 moff = bi.off + (u64)(m.p - b);
        for (u32 k = 0; k < N && !m.err; k++) {
            t.ch_msg_off[bi.ch0 + k] = moff;
            moff += t.ch_msg_len[bi.ch0 + k];
            m.skip(t.ch_msg_len[bi.ch0 + k]);
        }
        if (m.err || !m.empty()) err = err ? err : LB_ERR(DOC_ERR_DECODE);
    }
    // ---- keys
    {
        Cur k(b + bi.sec_off[3], bi.sec_len[3]);
        for (u32 q = 0; q < bi.n_keys; q++) {
            u64 len = k.varint();
            t.key_off[bi.key0 + q] = bi.off + (u64)(k.p - b);
            t.key_len[bi.key0 + q] = (u32)len;
            k.skip(len);
        }
        if (k.err) err = err ? err : LB_ERR(DOC_ERR_DECODE);
    }
    // ---- cids (row-wise postcard, field count 4)
    {
        Cur c(b + bi.sec_off[2], bi.sec_len[2]);
        (void)c.varint();
        for (u32 q = 0; q < bi.n_cids; q++) {
            if (c.varint() != 4) c.err = 1;
            u8 is_root = c.get();
            u8 type = c.get();
            u64 pidx = c.varint();
            i64 koc = c.zigzag();
            if (is_root > 1) c.err = 1;
            if (is_root) { if (koc < 0 || (u64)koc >= bi.n_keys) err = LB_ERR(DOC_ERR_CORRUPT); }
            else if (pidx >= bi.n_peers) err = LB_ERR(DOC_ERR_CORRUPT);
            t.cid_root[bi.cid0 + q] = is_root;
            t.cid_type[bi.cid0 + q] = type;
            t.cid_peer_idx[bi.cid0 + q] = (u32)pidx;
            t.cid_koc[bi.cid0 + q] = (i32)koc;
        }
        if (c.err || !c.empty()) err = err ? err : LB_ERR(DOC_ERR_DECODE);
    }
    // ---- positions: expand the prefix-compressed fractional indexes into the pool (arena.rs:187-204)
    if (bi.n_pos) {
        const u8* pc[2];
        u32 pl[2];
        columnar_open(b + bi.sec_off[4], bi.sec_len[4], 2, pc, pl);
        RleCur pre(pc[0], pl[0], 1);
        Cur rest(pc[1], pl[1]);
        (void)rest.varint();
        u64 w = bi.posb0, last_off = 0;
        u32 last_len = 0;
        for (u32 q = 0; q < bi.n_pos; q++) {
            i64 common = 0;
            pre.next(&common);
            u32 len = (u32)rest.varint();
            if (rest.err || (u64)common > last_len || w + (u64)common + len > bi.posb0 + bi.pos_bytes) { err = err ? err : LB_ERR(DOC_ERR_DECODE); break; }
            for (u32 k = 0; k < (u32)common; k++) t.pos_pool[w + k] = t.pos_pool[last_off + k];
            for (u32 k = 0; k < len; k++) t.pos_pool[w + (u32)common + k] = rest.get();
            t.pos_off[bi.pos0 + q] = w;
            t.pos_len[bi.pos0 + q] = (u32)common + len;
            last_off = w;
            last_len = (u32)common + len;
            w += last_len;
        }
    }
    return err;
}

// ---- the rows, one COLUMN at a time: a thread has a single byte cursor alive at any moment, so its cache lines stay
// resident in L1 between windows (seven cursors 4 KB apart, all columns at once, thrash it), the loop bodies need a
// fraction of the registers, and consecutive stores of a thread fall into the same 32-byte sector back to back.  The
// values walk reads the kind / length / container of a row back from the tables the column passes just wrote
// (sequential per thread).
template <int MODE, class Emit>
__device__ __forceinline__ u32 column_pass(const u8* col, u32 len, u32 n, Emit emit) {   // returns rows emitted, ~0u on malformed input
    RleCur c(col, len, MODE);
    i64 acc = 0;
    u32 r = 0;
    for (; r < n; r++) {
        i64 v;
        if (!c.next(&v)) break;
        if (MODE == 2) { acc += v; v = acc; }
        emit(r, v);
    }
    if (c.c.err) return 0xFFFFFFFFu;
    i64 extra;
    if (r == n && c.next(&extra)) return 0xFFFFFFFFu;   // more rows than announced
    return r;
}
__device__ inline u32 decode_block_rows_cols(const u8* b, const BlockInfo& bi, const BatchTables& t, u32 err, u32* n_maps_out) {
    const u32 N = bi.n_changes, R = bi.n_ops;
    // ---- delete start ids
    if (bi.sec_len[6]) {
        const u8* col[3];
        u32 cl[3];
        if (!columnar_open(b + bi.sec_off[6], bi.sec_len[6], 3, col, cl)) err = err ? err : LB_ERR(DOC_ERR_DECODE);
        else {
            const u64 d0 = bi.del0;
            const u32 np = bi.n_peers;
            bool corrupt = false;
            u32 n0 = column_pass<2>(col[0], cl[0], bi.n_dels, [&](u32 r, i64 v) { if (v < 0 || (u64)v >= np) corrupt = true; t.del_peer_idx[d0 + r] = (u32)v; });
            u32 n1 = column_pass<2>(col[1], cl[1], bi.n_dels, [&](u32 r, i64 v) { t.del_counter[d0 + r] = (i32)v; });
            u32 n2 = column_pass<2>(col[2], cl[2], bi.n_dels, [&](u32 r, i64 v) { if (v == 0) corrupt = true; t.del_len[d0 + r] = (i32)v; });
            if (n0 != bi.n_dels || n1 != bi.n_dels || n2 != bi.n_dels) err = err ? err : LB_ERR(DOC_ERR_DECODE);
            else if (corrupt) err = err ? err : LB_ERR(DOC_ERR_CORRUPT);
        }
    } else if (bi.n_dels) err = err ? err : LB_ERR(DOC_ERR_DECODE);
    // ---- ops columns
    const u8* col[4];
    u32 cl[4];
    columnar_open(b + bi.sec_off[5], bi.sec_len[5], 4, col, cl);   // (validated by the count pass)
    const u64 r0 = bi.op0;
    {
        const u32 nc = bi.n_cids;
        bool corrupt = false;
        u32 n0 = column_pass<2>(col[0], cl[0], R, [&](u32 r, i64 v) { if (v < 0 || (u64)v >= nc) { corrupt = true; v = 0; } t.op_cid[r0 + r] = (u32)v; });
        u32 n1 = column_pass<2>(col[1], cl[1], R, [&](u32 r, i64 v) { t.op_prop[r0 + r] = (i32)v; });
        u32 n2 = column_pass<0>(col[2], cl[2], R, [&](u32 r, i64 v) { t.op_vtype[r0 + r] = (u8)v; });
        // lengths: counters and the change of every row fall out of the same pass
        i32 counter = (i32)bi.counter_start;
        u32 change = 0, ch_first_row = 0;
        i32 next_boundary = (i32)bi.counter_start + (i32)t.ch_len[bi.ch0];
        t.ch_op0[bi.ch0] = r0;
        bool straddle = false;
        u32 n3 = column_pass<1>(col[3], cl[3], R, [&](u32 r, i64 v) {
            if (v <= 0 || v > 0x7FFFFFFF || change >= N) { corrupt = true; v = 1; }
            t.op_len[r0 + r] = (u32)v;
            t.op_counter[r0 + r] = counter;
            t.op_change[r0 + r] = (u32)(bi.ch0 + (change < N ? change : N - 1));
            counter += (i32)v;
            if (counter > next_boundary) straddle = true;
            if (counter == next_boundary && change < N) {
                t.ch_nops[bi.ch0 + change] = r + 1 - ch_first_row;
                change++;
                ch_first_row = r + 1;
                if (change < N) { t.ch_op0[bi.ch0 + change] = r0 + r + 1; next_boundary += (i32)t.ch_len[bi.ch0 + change]; }
            }
        });
        if (n0 != R || n1 != R || n2 != R || n3 != R) err = err ? err : LB_ERR(DOC_ERR_DECODE);
        else if (corrupt || straddle || change != N || counter != (i32)(bi.counter_start + bi.counter_len)) err = err ? err : LB_ERR(DOC_ERR_CORRUPT);
    }
    if (err) return err;
    // ---- values walk
    Cur v(b + bi.sec_off[7], bi.sec_len[7]);
    u32 ndel = 0, ntree = 0, n_maps = 0;
    for (u32 r = 0; r < R; r++) {
        const u64 row = r0 + r;
        const u8 vt = t.op_vtype[row];
        // (that a List insert carries exactly `len` items is checked row-parallel by k_op_classify: here it would cost
        //  two dependent table reads per row)
        const u8* v0 = v.p;
        u32 aux_idx = 0xFFFFFFFFu;
        if (vt == VK_RAW_TREE_MOVE) {
            u64 sp = v.varint(), sc = v.varint(), pi = v.varint();
            u8 pn = v.get();
            u64 pp = 0, pcn = 0;
            if (!pn) { pp = v.varint(); pcn = v.varint(); }
            if (ntree >= bi.n_tree || sp >= bi.n_peers || (!pn && pp >= bi.n_peers) || sc > 0x7FFFFFFFull || pcn > 0x7FFFFFFFull) { err = LB_ERR(DOC_ERR_CORRUPT); break; }
            u8 pk = pn ? TRP_ROOT : TRP_NODE;
            if (!pn && t.peer_id[bi.peer0 + (u32)pp] == DELETED_ROOT_PEER && (i32)pcn == DELETED_ROOT_CTR) pk = TRP_DELETED;
            if (pk != TRP_DELETED && pi >= bi.n_pos) { err = LB_ERR(DOC_ERR_CORRUPT); break; }
            u64 ti = bi.tr0 + ntree++;
            t.tr_target_peer[ti] = (u32)sp;
            t.tr_target_ctr[ti] = (i32)sc;
            t.tr_parent_kind[ti] = pk;
            t.tr_parent_peer[ti] = (u32)pp;
            t.tr_parent_ctr[ti] = (i32)pcn;
            t.tr_pos[ti] = pk == TRP_DELETED ? 0xFFFFFFFFu : (u32)(bi.pos0 + pi);
            aux_idx = (u32)ti;
        } else {
            skip_value(v, vt, &n_maps);
            if (v.err == CUR_ERR_DEEP) { err = LB_ERR(DOC_ERR_UNSUPPORTED); break; }
        }
        t.op_val_off[row] = bi.off + (u64)(v0 - b);
        t.op_val_len[row] = (u32)(v.p - v0);
        if (vt == VK_DELETE_SEQ) aux_idx = (u32)(bi.del0 + ndel++);
        t.op_del[row] = aux_idx;
    }
    if (!err && (v.err || !v.empty())) err = LB_ERR(DOC_ERR_DECODE);
    if (!err && (ndel != bi.n_dels || ntree != bi.n_tree)) err = LB_ERR(DOC_ERR_CORRUPT);
    *n_maps_out = n_maps;
    return err;
}

__device__ inline void decode_block_fail(const BlockInfo& bi, u64 i, const BatchTables& t, BlockInfo* blocks, u32 err) {
    {
        // row-parallel kernels find their document through op_change: every row of a failed block must point
        // at one of the block's own changes, whatever the walk above managed to write
        for (u32 r = 0; r < bi.n_ops; r++) t.op_change[bi.op0 + r] = (u32)bi.ch0;
        for (u32 k = 0; k < bi.n_changes; k++) t.ch_block[bi.ch0 + k] = (u32)i;
        blocks[i].err = err;
    }
}

// thread per block, one column at a time
__global__ void k_block_decode_cols(const u8* __restrict__ bytes, BlockInfo* __restrict__ blocks, u64 n_blocks, const __grid_constant__ BatchTables t) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_blocks) return;
    BlockInfo bi = blocks[i];
    if (bi.err) return;
    const u8* b = bytes + bi.off;
    u32 n_maps = 0;
    u32 err = decode_block_small(b, bi, i, t);
    err = decode_block_rows_cols(b, bi, t, err, &n_maps);
    blocks[i].n_value_maps = n_maps;
    if (err) decode_block_fail(bi, i, t, blocks, err);
}
