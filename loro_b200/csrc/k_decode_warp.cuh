// loro_b200 -- phase 2, warp per change block: the block is staged in shared memory by one bulk asynchronous copy
// (TMA 1-D: cp.async.bulk + mbarrier), its columns are expanded lane-parallel and written as consecutive rows.
//
// Replaces the same reference code as k_decode.cuh (block_encode.rs:527-659, serde_columnar 0.3.14 AnyRle / DeltaRle,
// encoding/value.rs:603-700); what changes is the shape of the work:
//   * DRAM sees one aligned bulk read of the block instead of 8-byte windows scattered over seven cursors
//     (which multiply the DRAM traffic over the algorithmic bytes);
//   * AnyRle columns: the warp walks the SEGMENTS (few: runs dominate) and expands each one over the lanes -- a run is
//     arithmetic (value, or acc + delta * k for DeltaRle), a literal segment is cut into varints by a ballot over the
//     continuation bits of 32 bytes at a time, lane j decoding the j-th varint, DeltaRle finishing with a warp scan;
//   * the values stream is a chain (the next value starts where this one ends).  Almost every block carries one
//     kind of value with a payload (LoroValue for List/Map documents, Str for Text, RawTreeMove for trees), so the
//     chain is a function of the byte position alone: every lane takes a chunk of the section and computes, backwards,
//     "a value starting at p leaves my chunk at exit(p) after cnt(p) values"; 32 table look-ups stitch the chunks
//     together, and each lane then walks its own chunk from its true entry.  Rows pick their value by rank;
//   * every SoA table is written with consecutive lanes on consecutive rows.
// Anything the fast path does not cover (a block larger than the staging buffer, two kinds of payload in one block,
// nested values, a values section beyond the table, malformed input) is handed to decode_block_rows_cols on one lane --
// the default decoder's row code: it rewrites the same rows and produces the precise error code, so the fast path never
// has to explain a failure.  Like the default decoder, it leaves the check that a List insert carries exactly `len`
// items to k_op_classify, which runs after every decoder; a block that fails it fails its document there.
#pragma once
#include "k_decode.cuh"

#define DW_WARPS 4
#define DW_BYTES 8192      // staged bytes per warp (block + 16-byte alignment slack)
#define DW_VALS 4608       // values-section bytes covered by the chain tables (32 chunks of 144)
#define DW_BAD 0xFFFFu

struct DwWarp {
    alignas(16) u8 bytes[DW_BYTES];
    u16 tab[DW_VALS];      // per position: (exit - chunk_end) << 8 | values inside the chunk ; later: rank -> position
    alignas(8) u64 bar;
    u32 pad_[2];
};

__device__ __forceinline__ int nth_set_bit(unsigned m, int n) {   // position of the n-th (0-based) set bit of m
#ifdef LB_SIMT_EMU
    for (int i = 0; i < 32; i++) if ((m >> i) & 1) { if (n == 0) return i; n--; }
    return 32;
#else
    return (int)__fns(m, 0, n + 1);
#endif
}
__device__ __forceinline__ i64 warp_incl_scan64(i64 v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        i64 t = __shfl_up_sync(LB_FULL, v, d);
        if (lane >= d) v += t;
    }
    return v;
}
// low 64 bits of the varint in s[a..e] (e = its last byte)
__device__ __forceinline__ u64 varint_at(const u8* s, u32 a, u32 e) {
    u64 v = 0;
    int sh = 0;
    for (u32 q = a; q <= e; q++) { if (sh < 64) v |= (u64)(s[q] & 0x7f) << sh; sh += 7; }
    return v;
}

// ---- lane-parallel expansion of one AnyRle column.  MODE 0: raw bytes, 1: varints, 2: zigzag deltas accumulated
// (DeltaRle).  emit(row, value) is called with consecutive rows on consecutive lanes.  Returns the number of rows;
// *bad is set when the column is malformed or longer than max_rows.
template <int MODE, class Emit>
__device__ inline u32 warp_expand_column(const u8* col, u32 len, u32 max_rows, int lane, Emit emit, bool* bad) {
    u32 pos = 0, row = 0;
    i64 acc = 0;
    while (pos < len) {
        // segment header (uniform): zigzag varint
        u64 h = 0;
        int sh = 0;
        bool ok = false;
        for (int q = 0; q < 10 && pos < len; q++) { u8 c = col[pos++]; h |= (u64)(c & 0x7f) << sh; sh += 7; if (!(c & 0x80)) { ok = true; break; } }
        i64 sl = (i64)(h >> 1) ^ -(i64)(h & 1);
        if (!ok || sl == 0) { *bad = true; return row; }
        if (sl > 0) {
            i64 val;
            if (MODE == 0) { if (pos >= len) { *bad = true; return row; } val = col[pos++]; }
            else {
                u64 v = 0;
                sh = 0;
                ok = false;
                for (int q = 0; q < 19 && pos < len; q++) { u8 c = col[pos++]; if (sh < 64) v |= (u64)(c & 0x7f) << sh; sh += 7; if (!(c & 0x80)) { ok = true; break; } }
                if (!ok) { *bad = true; return row; }
                val = MODE == 2 ? ((i64)(v >> 1) ^ -(i64)(v & 1)) : (i64)v;
            }
            u64 n = (u64)sl;
            if (n > (u64)(max_rows - row)) { *bad = true; return row; }
            for (u32 k = (u32)lane; k < (u32)n; k += 32) emit(row + k, MODE == 2 ? acc + val * (i64)(k + 1) : val);
            if (MODE == 2) acc += val * (i64)n;
            row += (u32)n;
        } else {
            u64 n64 = (u64)(-sl);
            if (n64 > (u64)(max_rows - row)) { *bad = true; return row; }
            u32 n = (u32)n64;
            if (MODE == 0) {
                if (n > len - pos) { *bad = true; return row; }
                for (u32 k = (u32)lane; k < n; k += 32) emit(row + k, (i64)col[pos + k]);
                pos += n;
                row += n;
            } else {
                u32 remaining = n;
                while (remaining) {
                    u32 avail = len - pos < 32 ? len - pos : 32;
                    u8 c = (u32)lane < avail ? col[pos + lane] : 0x80;
                    unsigned term = __ballot_sync(LB_FULL, (u32)lane < avail && !(c & 0x80));
                    u32 cntv = (u32)__popc(term);
                    if (cntv == 0) { *bad = true; return row; }   // truncated, or a varint longer than 32 bytes
                    if (cntv > remaining) cntv = remaining;
                    i64 v = 0;
                    if ((u32)lane < cntv) {
                        int e = nth_set_bit(term, lane);
                        int a = lane == 0 ? 0 : nth_set_bit(term, lane - 1) + 1;
                        if (e - a >= 19) *bad = true;
                        u64 raw = varint_at(col + pos, (u32)a, (u32)e);
                        v = MODE == 2 ? ((i64)(raw >> 1) ^ -(i64)(raw & 1)) : (i64)raw;
                    }
                    if (MODE == 2) {
                        v = warp_incl_scan64((u32)lane < cntv ? v : 0, lane) + acc;
                        acc = __shfl_sync(LB_FULL, v, (int)cntv - 1);
                    }
                    if ((u32)lane < cntv) emit(row + (u32)lane, v);
                    pos += (u32)nth_set_bit(term, (int)cntv - 1) + 1;
                    row += cntv;
                    remaining -= cntv;
                }
            }
        }
    }
    return row;
}

// ---- length of the value of kind `vt` that starts at s[p] (n = section bytes), 0 when it is not a plain value the
// fast path handles (nested lists / maps, more than 8 list items, longer than 255 bytes, out of bounds)
__device__ __forceinline__ u32 dw_varint_len(const u8* s, u32 p, u32 n, u64* out) {
    u64 v = 0;
    int sh = 0;
    for (u32 q = 0; q < 10 && p + q < n; q++) {
        u8 c = s[p + q];
        v |= (u64)(c & 0x7f) << sh;
        sh += 7;
        if (!(c & 0x80)) { *out = v; return q + 1; }
    }
    return 0;
}
__device__ inline u32 dw_scalar_len(const u8* s, u32 p, u32 n) {   // LoroValue scalar incl. its kind byte
    if (p >= n) return 0;
    u8 k = s[p];
    u64 v;
    switch (k) {
        case 0: case 1: case 2: return 1;
        case 3: { u32 l = dw_varint_len(s, p + 1, n, &v); return l ? 1 + l : 0; }   // SLEB128: same continuation bits
        case 4: return p + 9 <= n ? 9 : 0;
        case 5: case 6: { u32 l = dw_varint_len(s, p + 1, n, &v); if (!l || v > 255) return 0; return 1 + l + (u32)v; }
        case 9: return p + 2 <= n ? 2 : 0;
        default: return 0;
    }
}
__device__ inline u32 dw_value_len(const u8* s, u32 p, u32 n, u8 vt) {
    u32 L = 0;
    u64 v;
    switch (vt) {
        case VK_LORO_VALUE: {
            if (p >= n) return 0;
            if (s[p] != 7) { L = dw_scalar_len(s, p, n); break; }
            u32 l = dw_varint_len(s, p + 1, n, &v);
            if (!l || v > 8) return 0;
            L = 1 + l;
            for (u32 q = 0; q < (u32)v; q++) { u32 e = dw_scalar_len(s, p + L, n); if (!e) return 0; L += e; }
            break;
        }
        case VK_STR: case VK_BINARY: { u32 l = dw_varint_len(s, p, n, &v); if (!l || v > 255) return 0; L = l + (u32)v; break; }
        case VK_I64: case VK_DELTA_INT: L = dw_varint_len(s, p, n, &v); break;
        case VK_F64: L = 8; break;
        case VK_RAW_TREE_MOVE: {
            for (int q = 0; q < 3; q++) { u32 l = dw_varint_len(s, p + L, n, &v); if (!l) return 0; L += l; }
            if (p + L >= n) return 0;
            u8 pn = s[p + L];
            L += 1;
            if (!pn) for (int q = 0; q < 2; q++) { u32 l = dw_varint_len(s, p + L, n, &v); if (!l) return 0; L += l; }
            break;
        }
        default: return 0;
    }
    return (L == 0 || L > 255 || p + L > n) ? 0 : L;
}
__device__ __forceinline__ bool dw_zero_len_kind(u8 vt) {
    return vt == VK_NULL || vt == VK_TRUE || vt == VK_FALSE || vt == VK_DELETE_ONCE || vt == VK_DELETE_SEQ;
}

// ---- the rows of a staged block, lane-parallel.  false = not covered (or malformed): the caller runs the
// single-lane decoder, which rewrites every row.
__device__ inline bool dw_rows_fast(const u8* b, const BlockInfo& bi, const BatchTables& t, u16* tab, int lane) {
    bool bad = false;
    const u32 R = bi.n_ops;
    // ---- delete start ids: three DeltaRle columns
    if (bi.n_dels) {
        const u8* col[3];
        u32 cl[3];
        if (!bi.sec_len[6] || !columnar_open(b + bi.sec_off[6], bi.sec_len[6], 3, col, cl)) return false;
        const u64 d0 = bi.del0;
        const u32 np = bi.n_peers;
        u32 n0 = warp_expand_column<2>(col[0], cl[0], bi.n_dels, lane, [&](u32 r, i64 v) { if (v < 0 || (u64)v >= np) bad = true; t.del_peer_idx[d0 + r] = (u32)v; }, &bad);
        u32 n1 = warp_expand_column<2>(col[1], cl[1], bi.n_dels, lane, [&](u32 r, i64 v) { t.del_counter[d0 + r] = (i32)v; }, &bad);
        u32 n2 = warp_expand_column<2>(col[2], cl[2], bi.n_dels, lane, [&](u32 r, i64 v) { if (v == 0) bad = true; t.del_len[d0 + r] = (i32)v; }, &bad);
        if (n0 != bi.n_dels || n1 != bi.n_dels || n2 != bi.n_dels) bad = true;
    } else if (bi.sec_len[6]) return false;
    // ---- the four ops columns
    const u8* col[4];
    u32 cl[4];
    if (!columnar_open(b + bi.sec_off[5], bi.sec_len[5], 4, col, cl)) return false;
    const u64 r0 = bi.op0;
    {
        const u32 nc = bi.n_cids;
        u32 n0 = warp_expand_column<2>(col[0], cl[0], R, lane, [&](u32 r, i64 v) { if (v < 0 || (u64)v >= nc) { bad = true; v = 0; } t.op_cid[r0 + r] = (u32)v; }, &bad);
        u32 n1 = warp_expand_column<2>(col[1], cl[1], R, lane, [&](u32 r, i64 v) { t.op_prop[r0 + r] = (i32)v; }, &bad);
        u32 n2 = warp_expand_column<0>(col[2], cl[2], R, lane, [&](u32 r, i64 v) { t.op_vtype[r0 + r] = (u8)v; }, &bad);
        u32 n3 = warp_expand_column<1>(col[3], cl[3], R, lane, [&](u32 r, i64 v) { if (v <= 0 || v > 0x7FFFFFFF) { bad = true; v = 1; } t.op_len[r0 + r] = (u32)v; }, &bad);
        if (n0 != R || n1 != R || n2 != R || n3 != R) bad = true;
    }
    if (__any_sync(LB_FULL, bad)) return false;
    __syncwarp();
    // ---- counters, change of every row, first row of every change; kinds of value in the block
    const u32 N = bi.n_changes;
    const i32* chc = t.ch_counter + bi.ch0;   // written by lane 0 (decode_block_small) before the rows
    const i32 block_end = (i32)(bi.counter_start + bi.counter_len);
    u32 H = 0, n_del = 0, n_tree = 0, found = 0;
    u8 heavy = 0xFF;       // the one kind with a payload (0xFF: none yet)
    bool mixed = false;
    i64 carry = (i64)(i32)bi.counter_start;
    for (u32 g = 0; g < R; g += 32) {
        u32 r = g + (u32)lane;
        bool in = r < R;
        u32 ln = in ? t.op_len[r0 + r] : 0;
        i64 incl = warp_incl_scan64((i64)ln, lane);
        i64 ctr = carry + incl - ln;
        carry += __shfl_sync(LB_FULL, incl, 31);
        u8 vt = in ? t.op_vtype[r0 + r] : (u8)VK_NULL;
        bool z = dw_zero_len_kind(vt);
        unsigned hm = __ballot_sync(LB_FULL, in && !z);
        if (hm) {   // (uniform) the one kind with a payload, agreed on across the lanes
            u8 first = (u8)__shfl_sync(LB_FULL, (int)vt, __ffs(hm) - 1);
            if (heavy == 0xFF) heavy = first;
            if (__ballot_sync(LB_FULL, in && !z && vt != heavy)) mixed = true;
        }
        H += (u32)__popc(hm);
        n_del += (u32)__popc(__ballot_sync(LB_FULL, in && vt == VK_DELETE_SEQ));
        n_tree += (u32)__popc(__ballot_sync(LB_FULL, in && vt == VK_RAW_TREE_MOVE));
        bool starts = false;
        if (in) {
            if (ctr + ln > (i64)block_end) bad = true;
            // change holding this counter: last c with chc[c] <= ctr
            u32 lo = 0, hi = N;
            while (hi - lo > 1) { u32 mid = (lo + hi) >> 1; if ((i64)chc[mid] <= ctr) lo = mid; else hi = mid; }
            i64 next_b = lo + 1 < N ? (i64)chc[lo + 1] : (i64)block_end;
            if (ctr + ln > next_b) bad = true;           // a row never straddles a change boundary
            t.op_counter[r0 + r] = (i32)ctr;
            t.op_change[r0 + r] = (u32)(bi.ch0 + lo);
            if ((i64)chc[lo] == ctr) { t.ch_op0[bi.ch0 + lo] = r0 + r; starts = true; }
        }
        found += (u32)__popc(__ballot_sync(LB_FULL, starts));
    }
    if (__any_sync(LB_FULL, bad || mixed) || found != N || carry != (i64)block_end || n_del != bi.n_dels || n_tree != bi.n_tree) return false;
    __syncwarp();
    for (u32 c = (u32)lane; c < N; c += 32) {
        u64 nx = c + 1 < N ? t.ch_op0[bi.ch0 + c + 1] : r0 + R;
        t.ch_nops[bi.ch0 + c] = (u32)(nx - t.ch_op0[bi.ch0 + c]);
    }
    // ---- the values chain
    const u8* vs = b + bi.sec_off[7];
    const u32 V = bi.sec_len[7];
    if (V > DW_VALS || H > DW_VALS) return false;
    if (H == 0) { if (V != 0) return false; }
    else {
        const u32 CH = (V + 31) / 32;
        const u32 c_lo = (u32)lane * CH < V ? (u32)lane * CH : V, c_hi = c_lo + CH < V ? c_lo + CH : V;
        for (u32 p = c_hi; p-- > c_lo;) {
            u32 L = dw_value_len(vs, p, V, heavy);
            u16 e = DW_BAD;
            if (L) {
                u32 q = p + L;
                if (q >= c_hi) { if (q - c_hi <= 255) e = (u16)(((q - c_hi) << 8) | 1u); }
                else { u16 n = tab[q]; if (n != DW_BAD && (n & 0xFFu) < 254u) e = (u16)(n + 1u); }
            }
            tab[p] = e;
        }
        __syncwarp();
        // stitch the chunks: entry of chunk l+1 = where the chain leaves chunk l
        u32 entry = 0, hbase = 0, my_entry = 0, my_hbase = 0;
        bool broken = false;
        for (u32 l = 0; l < 32; l++) {
            u32 lo = l * CH < V ? l * CH : V, hi = lo + CH < V ? lo + CH : V;
            if ((u32)lane == l) { my_entry = entry; my_hbase = hbase; }
            if (entry < hi) {
                if (entry < lo) { broken = true; break; }
                u16 e = tab[entry];
                if (e == DW_BAD) { broken = true; break; }
                entry = hi + (e >> 8);
                hbase += e & 0xFFu;
            }
        }
        if (broken || entry != V || hbase != H) return false;
        __syncwarp();
        // every lane walks its own chunk from its entry: rank -> position
        {
            u32 p = my_entry, k = my_hbase;
            while (p < c_hi && p >= c_lo) {
                tab[k++] = (u16)p;
                p += dw_value_len(vs, p, V, heavy);
            }
        }
        __syncwarp();
    }
    // ---- rows: value extent, delete / tree index, per-kind checks
    const u64 voff = bi.off + bi.sec_off[7];
    u32 hc = 0, dc = 0, tc = 0;
    for (u32 g = 0; g < R; g += 32) {
        u32 r = g + (u32)lane;
        bool in = r < R;
        u8 vt = in ? t.op_vtype[r0 + r] : (u8)VK_NULL;
        bool hv = in && !dw_zero_len_kind(vt);
        unsigned hm = __ballot_sync(LB_FULL, hv), dm = __ballot_sync(LB_FULL, in && vt == VK_DELETE_SEQ),
                 tm = __ballot_sync(LB_FULL, in && vt == VK_RAW_TREE_MOVE);
        unsigned lt = (1u << lane) - 1u;
        u32 hi_ = hc + (u32)__popc(hm & lt);
        u32 p = hi_ < H ? tab[hi_] : V;
        u32 L = hv ? dw_value_len(vs, p, V, vt) : 0;
        if (in) {
            u32 aux = 0xFFFFFFFFu;
            if (vt == VK_DELETE_SEQ) aux = (u32)(bi.del0 + dc + (u32)__popc(dm & lt));
            if (vt == VK_LORO_VALUE && t.cid_type[bi.cid0 + t.op_cid[r0 + r]] == CT_LIST) {
                // a List insert carries LoroValue::List with exactly `len` items (outdated_encode_reordered.rs:246-262)
                u64 n_items = 0;
                u32 l = vs[p] == 7 ? dw_varint_len(vs, p + 1, V, &n_items) : 0;
                if (!l || n_items != (u64)t.op_len[r0 + r]) bad = true;
            }
            if (vt == VK_RAW_TREE_MOVE) {
                u64 sp, sc, pi, pp = 0, pcn = 0;
                u32 q = p;
                q += dw_varint_len(vs, q, V, &sp);
                q += dw_varint_len(vs, q, V, &sc);
                q += dw_varint_len(vs, q, V, &pi);
                u8 pn = vs[q++];
                if (!pn) { q += dw_varint_len(vs, q, V, &pp); q += dw_varint_len(vs, q, V, &pcn); }
                if (sp >= bi.n_peers || (!pn && pp >= bi.n_peers) || sc > 0x7FFFFFFFull || pcn > 0x7FFFFFFFull) bad = true;
                else {
                    u8 pk = pn ? TRP_ROOT : TRP_NODE;
                    if (!pn && t.peer_id[bi.peer0 + (u32)pp] == DELETED_ROOT_PEER && (i32)pcn == DELETED_ROOT_CTR) pk = TRP_DELETED;
                    if (pk != TRP_DELETED && pi >= bi.n_pos) bad = true;
                    u64 ti = bi.tr0 + tc + (u32)__popc(tm & lt);
                    t.tr_target_peer[ti] = (u32)sp;
                    t.tr_target_ctr[ti] = (i32)sc;
                    t.tr_parent_kind[ti] = pk;
                    t.tr_parent_peer[ti] = (u32)pp;
                    t.tr_parent_ctr[ti] = (i32)pcn;
                    t.tr_pos[ti] = pk == TRP_DELETED ? 0xFFFFFFFFu : (u32)(bi.pos0 + pi);
                    aux = (u32)ti;
                }
            }
            t.op_val_off[r0 + r] = voff + p;
            t.op_val_len[r0 + r] = L;
            t.op_del[r0 + r] = aux;
        }
        hc += (u32)__popc(hm);
        dc += (u32)__popc(dm);
        tc += (u32)__popc(tm);
    }
    return !__any_sync(LB_FULL, bad);
}

__global__ void __launch_bounds__(32 * DW_WARPS)
k_block_decode_warp(const u8* __restrict__ bytes, BlockInfo* __restrict__ blocks, u64 n_blocks, const __grid_constant__ BatchTables t) {
#ifdef LB_SIMT_EMU
    LB_DYN_SMEM(DwWarp, smem);
#else
    extern __shared__ __align__(16) u8 dw_smem_raw[];
    DwWarp* smem = (DwWarp*)dw_smem_raw;
#endif
    const int lane = threadIdx.x & 31;
    const u32 w = threadIdx.x >> 5;
    const u64 i = (u64)blockIdx.x * DW_WARPS + w;
    if (i >= n_blocks) return;
    BlockInfo bi = blocks[i];
    if (bi.err) return;
    DwWarp& S = smem[w];
    const u32 shift = (u32)(bi.off & 15);
    const u32 span = (shift + bi.len + 15u) & ~15u;
    const bool staged = span <= DW_BYTES;   // (uniform) a larger block is decoded from global memory by one lane
    const u8* b = bytes + bi.off;
    u32 err = 0, n_maps = 0;
    bool fast = false;
    if (staged) {
        // ---- stage the block: one bulk asynchronous copy, completion on the warp's mbarrier
#ifdef LB_SIMT_EMU
        for (u32 k = (u32)lane; k < span; k += 32) S.bytes[k] = bytes[bi.off - shift + k];
        __syncwarp();
#else
        {
            const u32 bar = (u32)__cvta_generic_to_shared(&S.bar);
            const u32 dst = (u32)__cvta_generic_to_shared(S.bytes);
            if (lane == 0) {
                asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(span) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dst), "l"(bytes + (bi.off - shift)), "r"(span), "r"(bar) : "memory");
            }
            __syncwarp();
            u32 done = 0;
            while (!done) {
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(done) : "r"(bar), "r"(0u) : "memory");
            }
        }
#endif
        b = S.bytes + shift;
        if (lane == 0) err = decode_block_small(b, bi, i, t);
        err = (u32)__shfl_sync(LB_FULL, (int)err, 0);
        __syncwarp();
        fast = !err && dw_rows_fast(b, bi, t, S.tab, lane);
        __syncwarp();
    }
    // one call site for the one-lane rows: with a second call of decode_block_rows_cols ptxas keeps one of them as a
    // real call, and the kernel drops to 80 registers and spills
    if (lane == 0) {
        if (!staged) err = decode_block_small(b, bi, i, t);
        if (!fast) err = decode_block_rows_cols(b, bi, t, err, &n_maps);
        atomicAdd(&t.dw_stats[fast ? 0 : staged ? 1 : 2], 1ull);
        blocks[i].n_value_maps = n_maps;
        if (err) decode_block_fail(bi, i, t, blocks, err);
    }
}
