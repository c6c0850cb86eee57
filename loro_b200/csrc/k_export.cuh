// loro_b200 -- phase 7: re-export of every document as a FastUpdates blob (ExportMode::all_updates).
//
// Replaces (reference, relative to crates/loro-internal/src):
//   encoding.rs:350-416 (export, header + xxHash32), encoding/fast_snapshot.rs:257-260 (body framing),
//   oplog/change_store.rs:494-576,711-764,1244-1291 (export_blocks_from -> a fresh store: block packing with
//     MAX_BLOCK_SIZE, ChangesBlock::push_change), change.rs:128-139,268-283 (estimate_storage_size,
//     can_merge_right), op.rs:143-148 + container/list/list_op.rs:189-278,381-434,516-658 (RleVec merge rules),
//   oplog/change_store/block_encode.rs:137-278 (encode_block), block_meta_encode.rs:13-88 (encode_changes),
//   encoding/arena.rs:103-147 (ContainerArena), serde_columnar 0.3.14 column encoders (BoolRle, AnyRle,
//   DeltaRle, DeltaOfDelta; SURVEY Appendix B).
//
// What the imported document's change store looks like is re-derived from the decoded tables:
//   A  (warp per change, 32 rows at a time) ops of each decoded change go through the RleVec merge
//      (block_encode.rs:651); a change whose size estimate exceeds one block is cut into segments
//      (split_change_then_insert, one lane), List / Text inserts that do not fit a block are themselves cut
//      (Op::slice) -- such a change is re-written as synthetic rows (thread per change);
//   B  (thread per document, per peer in id order) the segments enter the store in counter order
//      (ChangeStore::insert_change, merge_interval 0 for imports), and what comes out is pushed, as it completes,
//   C  into the fresh store export builds (export_blocks_from): same rules, freshly computed sizes.
// Only per-row flag bits (op start, segment start) and per-segment summaries are written; the merge decisions
// look at the boundary ops only.  A thread per output block then gathers its ops into scratch columns and
// encodes them once, into a staging slot sized from the block's rows and store estimate; the lengths it records
// place the block in its document's blob, and a warp per document assembles the blob from the staged pieces and the
// length prefixes.  A block that outgrows its slot is encoded again by the same code, into a slot of its exact size.
// Whether two neighbouring inserts merge depends on where their payloads landed in the importing document's
// arenas (arena.rs:237-263): values are adjacent when nothing else was allocated in between (decode order),
// strings additionally need the append-only buffer not to have been reallocated (capacity doubles from 32;
// restated from append-only-bytes 0.1.12, same model as the oracle, unpinned by reference tests).
// Values containing nested maps carry block-local key indices: xvalue_copy re-registers their keys in the output
// block.  Documents with MovableList, Counter or style ops are not covered (lb_doc_export_updates answers
// LB_ERR_UNSUPPORTED for them).  Pending changes stay out of the
// export but their payloads still count for the arena positions; a document built from several blobs sees them
// in import_batch's order (the host lays them out that way).
#pragma once
#include "lb_tables.cuh"

enum { XK_NONE = 0, XK_LIST = 1, XK_TEXT = 2, XK_DEL = 3, XK_MAPSET = 4, XK_MAPDEL = 5, XK_TREE = 6 };
#define LB_MAX_BLOCK_SIZE 4096   // change_store.rs:37
#define XF_HEAD 1u               // row starts a (merged) op
#define XF_SEG 2u                // row starts a segment of a split change

struct XDoc {          // per document
    u32 n_fc, n_mb;    // final changes, output blocks
    u32 flags;         // bit0: export unsupported for this document ; bit1: the document has movable-tree ops ;
                       // bit2: some value holds a nested map (its keys are indices into the block's key arena)
    u32 n_prank;       // distinct fractional indexes of the document (k_exp_posrank)
    u64 ob0;           // first output block (batch-wide)
    u64 scratch0;      // first scratch word of this doc's blocks
    u64 exp_off;       // offset of the blob in the export buffer
    u32 exp_len;
    u32 scratch_words;
    u64 stage0;        // first staging byte of this doc's blocks
    u64 ovf0;          // blocks of the documents before this one that outgrew their staging slot (scan)
    u64 restage0;      // first retry-slot byte of this doc's blocks that outgrew their staging slot (scan)
};
struct XBlock {        // one output block
    u32 doc;
    u32 fc0, fc1;      // final-change range (absolute indices into fc_*)
    u32 len;           // encoded bytes (without the ULEB length prefix)
    u32 sec_len[8];
    u32 col_len[9];    // ops columns 0-3, delete columns 4-6, position columns 7-8
    u64 off;           // offset of the block bytes inside the document's blob
    u64 scratch;       // scratch words of this block
    u32 n_rows, n_dels;            // scratch capacities: rows, delete ops
    u32 n_ops, n_del_ops, n_pos;   // after the gather: merged ops, merged deletes, positions
    u64 stage;         // staging slot: first byte, capacity; the block's pieces without their length prefixes
    u32 stage_cap;
    u32 ovf;           // 1 = the pieces did not fit the first slot: encoded again into a retry slot (k_exp_layout;
                       //     `stage` is then relative to the document's restage0)
};

// ---------------------------------------------------------------------------------------------- byte sink
struct XSink {
    u8* dst;   // bytes [0, cap) are stored; what lies beyond is only counted (cap = 0: a counting sink)
    u64 n, cap;
    __device__ __forceinline__ XSink(u8* d, u64 c) : dst(d), n(0), cap(c) {}
    // (plain byte stores: collecting eight bytes per store or reading the scratch columns through a four-word window
    //  adds instructions and registers to every byte of an encoder bound by dependent-load latency at 25 % occupancy)
    __device__ __forceinline__ void put(u8 c) { if (n < cap) dst[n] = c; n++; }
    __device__ __forceinline__ void varint(u64 v) { while (v >= 0x80) { put((u8)(v | 0x80)); v >>= 7; } put((u8)v); }
    __device__ __forceinline__ void zigzag(i64 v) { varint(((u64)v << 1) ^ (u64)(v >> 63)); }
    __device__ __forceinline__ void copy(const u8* s, u64 len) {
        if (n + len <= cap) {
            u8* d = dst + n;
            u64 i = 0;
            while (i < len && ((uintptr_t)(d + i) & 3)) { d[i] = s[i]; i++; }
            for (; i + 4 <= len; i += 4) {   // 4 independent byte loads, one aligned word store
                u32 w = (u32)s[i] | ((u32)s[i + 1] << 8) | ((u32)s[i + 2] << 16) | ((u32)s[i + 3] << 24);
                *(u32*)(d + i) = w;
            }
            for (; i < len; i++) d[i] = s[i];
        }
        n += len;
    }
};
__device__ __forceinline__ u32 varint_len(u64 v) { u32 k = 1; while (v >= 0x80) { v >>= 7; k++; } return k; }

// ---------------------------------------------------------------------------------------------- merge rules
struct XOp {   // one (possibly merged) op: the fields the merge rules and the encoder need
    u8 xk; u32 cidx; i32 ctr; u32 atoms; i32 prop; u32 f0, f1; i32 f2; u32 st0, nst;
    u32 g;   // TEXT: generation of the string arena buffer when the op's payload was allocated
    // LIST/TEXT: f0 = arena start, f1 = arena end (TEXT: bytes; f1 - f0 = payload bytes)
    // DEL: f0 = target peer (doc-level), f1 = lowest target counter, f2 = signed length
};
__device__ __forceinline__ u32 xop_estimate(const XOp& o) {   // list_op.rs:109-123, op/content.rs:70-77
    switch (o.xk) {
        case XK_LIST: return 4 * o.atoms;
        case XK_TEXT: return o.f1 - o.f0;
        case XK_DEL: return 8;
        case XK_TREE: return 8;        // op/content.rs:70-77
        default: return 3;
    }
}
// string arena generation: number of capacity doublings (from 32) needed to hold `end` bytes
__device__ __forceinline__ u32 str_gen(u32 end) {
    u32 k = 0;
    u64 cap = 32;
    while (cap < end) { cap <<= 1; k++; }
    return k;
}
// DeleteSpan helpers (list_op.rs:381-444); prop = pos, f2 = signed len, (f0, f1) = id_start
__device__ __forceinline__ bool d_bidi(const XOp& o) { return o.f2 == 1 || o.f2 == -1; }
__device__ __forceinline__ i64 d_start_pos(const XOp& o) { return o.f2 > 0 ? o.prop : (i64)o.prop + 1 + o.f2; }
__device__ __forceinline__ i64 d_next_pos(const XOp& o) { return o.f2 > 0 ? d_start_pos(o) : d_start_pos(o) - 1; }
__device__ __forceinline__ i64 d_prev_pos(const XOp& o) { return o.f2 > 0 ? o.prop : (i64)o.prop + 1; }
__device__ __forceinline__ i64 d_id_end(const XOp& o) { return (i64)(i32)o.f1 + (o.f2 < 0 ? -o.f2 : o.f2); }
__device__ inline bool xop_mergable(const XOp& a, const XOp& b) {   // op.rs:143-148 + list_op.rs:516-552
    if (a.ctr + (i32)a.atoms != b.ctr || a.cidx != b.cidx || a.xk != b.xk) return false;
    switch (a.xk) {
        case XK_LIST: return (i64)a.prop + a.atoms == b.prop && a.f1 == b.f0;
        case XK_TEXT: return (i64)a.prop + a.atoms == b.prop && a.f1 == b.f0 && a.g == b.g;
        case XK_DEL: {
            if (a.f0 != b.f0) return false;    // ids of different peers never line up
            bool ab = d_bidi(a), bb = d_bidi(b);
            i64 as = (i32)a.f1, bs = (i32)b.f1;
            if (ab && bb) return (a.prop == b.prop && as + 1 == bs) || ((i64)a.prop == (i64)b.prop + 1 && as == bs + 1);
            if (ab && !bb) {
                if (a.prop == d_prev_pos(b)) return b.f2 > 0 ? as + 1 == bs : as == d_id_end(b);
                return false;
            }
            if (!ab && bb) {
                if (d_next_pos(a) == b.prop) return a.f2 > 0 ? d_id_end(a) == bs : as == bs + 1;
                return false;
            }
            if (d_next_pos(a) == b.prop && (a.f2 > 0) == (b.f2 > 0)) return a.f2 > 0 ? d_id_end(a) == bs : as == d_id_end(b);
            return false;
        }
        default: return false;
    }
}
__device__ inline void xop_merge(XOp& a, const XOp& b) {
    switch (a.xk) {
        case XK_LIST: case XK_TEXT: a.f1 = b.f1; break;
        case XK_DEL: {   // list_op.rs:244-249, 398-434
            bool ab = d_bidi(a), bb = d_bidi(b);
            i32 as = (i32)a.f1, bs = (i32)b.f1;
            i32 nl;
            if (ab && bb) nl = a.prop == b.prop ? 2 : -2;
            else if (ab && !bb) nl = b.f2 + (b.f2 > 0 ? 1 : -1);
            else if (!ab && bb) nl = a.f2 + (a.f2 > 0 ? 1 : -1);
            else nl = a.f2 + b.f2;
            a.f1 = (u32)(as < bs ? as : bs);
            a.f2 = nl;
            break;
        }
        default: break;
    }
    a.atoms += b.atoms;
    a.nst += b.nst;
}

// one decoded row as an op (map keys and delete targets at document level): the resolving form walks the decode
// tables (container type, block key arena, delete table); k_exp_changes runs it once per row and leaves a 16-byte
// record, which is what every later pass loads (three independent loads per row instead of a chain)
__device__ inline XOp xop_resolve(const BatchTables& t, const DocInfo& di, u32 ch, u64 row, u32 astart) {
    XOp o;
    u8 kind = t.op_kind[row];
    o.cidx = t.op_cidx[row];
    o.ctr = t.op_counter[row];
    o.atoms = t.op_len[row];
    o.prop = t.op_prop[row];
    o.f0 = o.f1 = 0; o.f2 = 0; o.g = 0;
    o.st0 = (u32)row; o.nst = 1;
    switch (kind) {
        case OPK_SEQ_INS:
            if (t.dcont[di.cid0 + o.cidx].type == CT_TEXT) { o.xk = XK_TEXT; o.f0 = astart; o.f1 = o.f0 + t.r_bytes[row]; o.g = str_gen(o.f1); }
            else { o.xk = XK_LIST; o.f0 = astart; o.f1 = o.f0 + o.atoms; }
            break;
        case OPK_SEQ_DEL: {
            u32 dl = t.op_del[row];
            o.xk = XK_DEL; o.f0 = t.op_aux[row]; o.f1 = (u32)t.del_counter[dl]; o.f2 = t.del_len[dl];
            break;
        }
        case OPK_MAP_SET: case OPK_MAP_DEL:
            o.xk = kind == OPK_MAP_SET ? XK_MAPSET : XK_MAPDEL;
            o.prop = (i32)t.key_map[t.blocks[t.ch_block[ch]].key0 + (u32)o.prop];
            break;
        case OPK_TREE: o.xk = XK_TREE; o.prop = 0; o.f0 = t.op_del[row]; break;   // f0 = index into the tr_* tables
        default: o.xk = XK_NONE;
    }
    return o;
}
__device__ __forceinline__ uint4 xop_pack(const XOp& o) {
    uint4 r;
    r.x = (u32)o.xk | ((o.xk == XK_DEL && o.f2 < 0) ? 8u : 0u) | (o.cidx << 4);
    r.y = (u32)o.ctr;
    r.z = (u32)o.prop;
    r.w = o.xk == XK_DEL ? o.f1 : o.f0;
    return r;
}
// ---- row accessors: decoded rows [0, n_rows) and synthetic rows [n_rows, ...)
__device__ __forceinline__ uint4 xr_rec(const BatchTables& t, u64 row) { return (!t.has_syn || row < t.n_rows) ? t.x_rec[row] : t.s_rec[row - t.n_rows]; }
__device__ __forceinline__ u32 xr_len(const BatchTables& t, u64 row) { return (!t.has_syn || row < t.n_rows) ? t.op_len[row] : t.s_len[row - t.n_rows]; }
__device__ __forceinline__ u32 xr_bytes(const BatchTables& t, u64 row) { return (!t.has_syn || row < t.n_rows) ? t.r_bytes[row] : t.s_bytes[row - t.n_rows]; }
__device__ __forceinline__ u32 xr_aux(const BatchTables& t, u64 row) { return (!t.has_syn || row < t.n_rows) ? t.op_aux[row] : t.s_aux[row - t.n_rows]; }
__device__ __forceinline__ u8* xr_flagp(const BatchTables& t, u64 row) { return (!t.has_syn || row < t.n_rows) ? &t.r_flag[row] : &t.s_flag[row - t.n_rows]; }
__device__ __forceinline__ u8 xr_flag(const BatchTables& t, u64 row) { return *xr_flagp(t, row); }
// the rows of a change as the export sees them
__device__ __forceinline__ void change_rows(const BatchTables& t, u32 ch, u64* row0, u32* nr) {
    u32 ns = t.has_syn ? t.ch_syn[ch] : 0;
    if (ns) { *row0 = t.n_rows + t.ch_syn0[ch]; *nr = ns; }
    else { *row0 = t.ch_op0[ch]; *nr = t.ch_nops[ch]; }
}
// payload bytes a row contributes to the values section (items of a list insert, text bytes, a whole map value)
__device__ __forceinline__ void xr_payload(const BatchTables& t, u64 row, u32 xk, const u8** p, u32* n) {
    if (t.has_syn && row >= t.n_rows) { *p = t.bytes + t.s_voff[row - t.n_rows]; *n = t.s_vlen[row - t.n_rows]; return; }
    const u8* v = t.bytes + t.op_val_off[row];
    u32 vl = t.op_val_len[row];
    if (xk == XK_LIST) {            // `07` + item count (parsed, not assumed minimal)
        Cur c(v, vl);
        (void)c.get();
        (void)c.varint();
        *p = c.p;
        *n = (u32)c.left();
    } else if (xk == XK_TEXT) {     // byte length + bytes
        Cur c(v, vl);
        (void)c.varint();
        *p = c.p;
        *n = (u32)c.left();
    }
    else if (xk == XK_MAPSET) { *p = v; *n = vl; }
    else { *p = v; *n = 0; }
}
__device__ __forceinline__ XOp xop_from_row(const BatchTables& t, const DocInfo&, u32, u64 row) {
    uint4 r = xr_rec(t, row);
    XOp o;
    o.xk = (u8)(r.x & 7u);
    o.cidx = r.x >> 4;
    o.ctr = (i32)r.y;
    o.prop = (i32)r.z;
    o.atoms = xr_len(t, row);
    o.f0 = r.w; o.f1 = 0; o.f2 = 0; o.g = 0;
    o.st0 = (u32)row; o.nst = 1;
    if (o.xk == XK_LIST) o.f1 = o.f0 + o.atoms;
    else if (o.xk == XK_TEXT) { o.f1 = o.f0 + xr_bytes(t, row); o.g = (!t.has_syn || row < t.n_rows) ? str_gen(o.f1) : xr_aux(t, row); }
    else if (o.xk == XK_DEL) { o.f0 = xr_aux(t, row); o.f1 = r.w; o.f2 = (r.x & 8u) ? -(i32)o.atoms : (i32)o.atoms; }
    return o;
}
// byte offset of unicode scalar value k inside a UTF-8 payload of nb bytes holding n scalar values
__device__ inline u32 text_byte_index(const u8* p, u32 nb, u32 n, u32 k) {
    if (nb == n || k == 0) return k < nb ? k : nb;   // ASCII
    u32 i = 0, ch = 0;
    while (i < nb && ch < k) {
        i++;
        while (i < nb && (p[i] & 0xC0) == 0x80) i++;
        ch++;
    }
    return i;
}
// payload of a row without its first `skip` atoms (list items / unicode scalar values)
__device__ inline void xr_payload_skip(const BatchTables& t, u64 row, u32 xk, u32 skip, const u8** p, u32* n) {
    xr_payload(t, row, xk, p, n);
    if (!skip) return;
    u32 off = 0;
    if (xk == XK_TEXT) off = text_byte_index(*p, *n, xr_len(t, row), skip);
    else if (xk == XK_LIST) {
        Cur c(*p, *n);
        for (u32 k = 0; k < skip && !c.err; k++) { u8 kk = c.get(); skip_loro_value_content(c, kk, nullptr); }
        off = (u32)(c.p - *p);
    }
    *p += off;
    *n -= off;
}
// ... and without its last `tail` atoms too, given the payload of its `atoms` atoms after the skip
__device__ inline void xr_payload_drop_tail(u32 xk, u32 atoms, u32 tail, const u8* p, u32* n) {
    if (xk == XK_TEXT) *n = text_byte_index(p, *n, atoms, atoms - tail);
    else if (xk == XK_LIST) {
        Cur c(p, *n);
        for (u32 k = 0; k < atoms - tail && !c.err; k++) { u8 kk = c.get(); skip_loro_value_content(c, kk, nullptr); }
        *n = (u32)(c.p - p);
    }
}
// Op::slice(skip, len) of the op made from `row` (op.rs:161-172, list_op.rs:603-658, 251-278, 436-444)
__device__ inline void xop_slice_front(const BatchTables& t, XOp& o, u64 row, u32 skip) {
    if (!skip) return;
    switch (o.xk) {
        case XK_LIST: o.prop += (i32)skip; o.f0 += skip; break;
        case XK_TEXT: {
            const u8* pp; u32 pn;
            xr_payload(t, row, XK_TEXT, &pp, &pn);
            o.prop += (i32)skip;
            o.f0 += text_byte_index(pp, pn, o.atoms, skip);
            break;
        }
        case XK_DEL:
            if (o.f2 > 0) { o.f1 += skip; o.f2 -= (i32)skip; }
            else { o.prop -= (i32)skip; o.f2 += (i32)skip; }
            break;
        default: return;   // one-atom ops are never cut
    }
    o.ctr += (i32)skip;
    o.atoms -= skip;
}
// Op::slice(0, atoms - tail) of an op whose last row is `row` (read for Text only): list_op.rs:251-278, 436-444
__device__ inline void xop_slice_back(const BatchTables& t, XOp& o, u64 row, u32 tail) {
    if (!tail) return;
    switch (o.xk) {
        case XK_LIST: o.f1 -= tail; break;
        case XK_TEXT: {
            const u8* pp; u32 pn;
            xr_payload(t, row, XK_TEXT, &pp, &pn);
            const u32 ra = xr_len(t, row);
            o.f1 -= pn - text_byte_index(pp, pn, ra, ra - tail);
            break;
        }
        case XK_DEL:   // a reversed span keeps its position and loses its lowest ids
            if (o.f2 > 0) o.f2 -= (i32)tail;
            else { o.f1 += tail; o.f2 += (i32)tail; }
            break;
        default: return;   // one-atom ops are never cut
    }
    o.atoms -= tail;
}

// ---------------------------------------------------------------------------------------------- X1: arenas
// The importing document allocates arena space while it decodes (block_encode.rs:619-657): the position of a row's
// payload is the sum over the rows decoded before it.  Changes are numbered in decode order, so: per-change sums
// (warp per change), one scan over the changes, and k_exp_changes hands out the row positions.
//
// Every decoded op allocates, applied or still pending (decode precedes the pending check: encoding.rs:232-270), so
// the arena a row allocates from is taken from (container type, value kind), not from op_kind.
enum { XA_NONE = 0, XA_VAL = 1, XA_STR = 2 };
#define XCH_TPB 128   // CTA of the warp-per-change kernels (k_exp_arena, k_exp_changes)
__device__ __forceinline__ u32 xr_arena(const BatchTables& t, const DocInfo& di, u64 row) {
    u8 ctype = t.dcont[di.cid0 + t.op_cidx[row]].type;
    u8 vt = t.op_vtype[row];
    if (ctype == CT_TEXT && vt == VK_STR) return XA_STR;
    if (ctype == CT_LIST && vt == VK_LORO_VALUE) return XA_VAL;
    return XA_NONE;
}
__device__ __forceinline__ u32 warp_sum_u32(u32 v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(LB_FULL, v, d);
    return v;
}
__device__ __forceinline__ u32 warp_incl_scan_u32(u32 v, u32 lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        u32 x = __shfl_up_sync(LB_FULL, v, d);
        if (lane >= (u32)d) v += x;
    }
    return v;
}
__global__ void k_exp_init(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    XDoc x;
    memset(&x, 0, sizeof(x));
    if (di.code == DOC_OK) {
        if (di.has_unsupported & 0x7FFFFFFFu) x.flags |= 1;
        if (di.has_tree) x.flags |= 2;
        for (u32 b = di.b0; b < di.b1; b++)
            if (t.blocks[b].n_value_maps) x.flags |= 4;   // payloads with nested maps: key indices are re-registered
    }
    t.xdoc[d] = x;
}
// warp per change: the lanes take 32 consecutive rows at a time (a change holds some hundreds of rows; a thread per
// change put the lanes of a warp hundreds of rows apart, one sector per lane for every column it loads)
__global__ void k_exp_arena(u64 n_changes, const __grid_constant__ BatchTables t, const DocInfo* __restrict__ docs) {
    const u64 ch = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const u32 lane = threadIdx.x & 31;
    if (ch >= n_changes) return;   // (whole warps)
    const BlockInfo& sb = t.blocks[t.ch_block[ch]];
    const DocInfo& di = docs[sb.doc];
    u32 vals = 0, strs = 0;
    if (di.code == DOC_OK) {
        const u64 r0 = t.ch_op0[ch];
        const u32 nr = t.ch_nops[ch];
        for (u32 r = lane; r < nr; r += 32) {
            const u64 row = r0 + r;
            const u32 a = xr_arena(t, di, row);
            if (a == XA_STR) {
                Cur c(t.bytes + t.op_val_off[row], t.op_val_len[row]);
                u32 n = (u32)c.varint();
                t.r_bytes[row] = n;
                strs += n;
            } else if (a == XA_VAL) vals += t.op_len[row];
        }
    }
    vals = warp_sum_u32(vals);
    strs = warp_sum_u32(strs);
    if (lane == 0) {
        t.ch_aval[ch] = vals;
        t.ch_astr[ch] = strs;
    }
}

// ---------------------------------------------------------------------------------------------- A: per change
// split_change_then_insert (change_store.rs:913-1000) for one change whose estimate exceeds a block: walks the
// merged ops, cuts List / Text inserts that do not fit (Op::slice) and reports every piece -- atoms [a,b) of source
// row `row`, whether it starts an op and whether it starts a segment -- to `emit`.
struct XSplit { u32 nseg, nsyn; bool sliced; };
template <class Emit>
__device__ inline XSplit split_change(const BatchTables& t, const DocInfo& di, u32 ch, u64 r0, u32 nr, u32 est0, Emit emit) {
    XSplit out;
    out.nseg = 0; out.nsyn = 0; out.sliced = false;
    u64 est = est0;
    bool has_ops = false, seg_next = true;
    u32 r = 0;
    while (r < nr) {
        // the merged op: rows [r, r1)
        XOp o = xop_from_row(t, di, ch, r0 + r);
        u32 r1 = r + 1;
        while (r1 < nr && !(t.r_flag[r0 + r1] & XF_HEAD)) { xop_merge(o, xop_from_row(t, di, ch, r0 + r1)); r1++; }
        const bool ins = o.xk == XK_LIST || o.xk == XK_TEXT;
        const u32 total_bytes = o.xk == XK_TEXT ? o.f1 - o.f0 : 0;
        u32 done = 0, done_bytes = 0;          // atoms / text bytes of this op already handed out
        u32 cr = r, coff = 0;                  // source row and atom offset where the rest of the op starts
        // hand out the next `count` atoms as one op
        auto piece = [&](u32 count) {
            bool head = true;
            while (count) {
                u32 ra = t.op_len[r0 + cr];
                u32 take = ra - coff < count ? ra - coff : count;
                u32 pb = 0;
                if (o.xk == XK_TEXT) {
                    const u8* pp; u32 pn;
                    xr_payload(t, r0 + cr, XK_TEXT, &pp, &pn);
                    pb = text_byte_index(pp, pn, ra, coff + take) - text_byte_index(pp, pn, ra, coff);
                }
                emit(r0 + cr, coff, coff + take, head, head && seg_next);
                if (head && seg_next) { out.nseg++; seg_next = false; }
                out.nsyn++;
                head = false;
                done += take;
                done_bytes += pb;
                count -= take;
                coff += take;
                if (coff == ra) { cr++; coff = 0; }
            }
            has_ops = true;
        };
        auto flush = [&]() { if (has_ops) { seg_next = true; est = 4; has_ops = false; } };
        auto rest_size = [&]() -> u64 { return o.xk == XK_TEXT ? total_bytes - done_bytes : (o.xk == XK_LIST ? 4ull * (o.atoms - done) : xop_estimate(o)); };
        if (rest_size() >= (u64)LB_MAX_BLOCK_SIZE - est) flush();
        bool consumed = false;
        while (true) {
            u64 room = (u64)LB_MAX_BLOCK_SIZE - est;
            if (rest_size() <= room || !ins) break;
            u32 rem = o.atoms - done;
            u64 end = o.xk == XK_TEXT ? (room < rem ? room : rem) : (room / 4 < rem ? room / 4 : rem);
            if (end == 0) break;
            out.sliced = true;
            piece((u32)end);
            flush();
            if (done >= o.atoms) { consumed = true; break; }
        }
        if (!consumed) {
            if (!ins) {
                // ops that are never cut are copied row by row (a merged delete span keeps its rows)
                est += rest_size();
                if (est > LB_MAX_BLOCK_SIZE && has_ops) flush();
                for (u32 q = r; q < r1; q++) {
                    bool head = q == r;
                    emit(r0 + q, 0, t.op_len[r0 + q], head, head && seg_next);
                    if (head && seg_next) { out.nseg++; seg_next = false; }
                    out.nsyn++;
                }
                has_ops = true;
            } else {
                est += rest_size();
                if (est > LB_MAX_BLOCK_SIZE && has_ops) flush();
                piece(o.atoms - done);
            }
        }
        r = r1;
    }
    return out;
}

// one summary record per segment of a change whose rows (decoded or synthetic) carry XF_HEAD / XF_SEG
__device__ inline void segment_summaries(const BatchTables& t, const DocInfo& di, u32 ch) {
    u64 row0;
    u32 nr;
    change_rows(t, ch, &row0, &nr);
    u64 sg_next = t.n_changes + t.ch_seg0[ch];
    u64 sg = ch;
    u32 r = 0, from = 0;
    while (r < nr) {
        u32 r_start = r, est = 0, nm = 0, ndel = 0, atoms = 0, last_head = r;
        do {
            XOp o = xop_from_row(t, di, ch, row0 + r);
            last_head = r;
            u32 r1 = r + 1;
            while (r1 < nr && !(xr_flag(t, row0 + r1) & (XF_HEAD | XF_SEG))) { xop_merge(o, xop_from_row(t, di, ch, row0 + r1)); r1++; }
            est += xop_estimate(o);
            nm++;
            ndel += o.xk == XK_DEL;
            atoms += o.atoms;
            r = r1;
        } while (r < nr && !(xr_flag(t, row0 + r) & XF_SEG));
        t.sg_src[sg] = ch; t.sg_r0[sg] = r_start; t.sg_from[sg] = from; t.sg_atoms[sg] = atoms; t.sg_est[sg] = est;
        t.sg_nmops[sg] = nm; t.sg_ndel[sg] = ndel; t.sg_nrows[sg] = r - r_start; t.sg_last_head[sg] = last_head; t.sg_skip[sg] = 0;
        from += atoms;
        sg = sg_next++;
    }
}

// XF_HEAD (the RleVec merge inside a change) from neighbouring rows.  The serial rule keeps `back`, the merged op
// the previous row ended in, and row r merges when xop_mergable(back, row r).  For List / Text a pairwise test of
// row r against row r - 1 decides the same thing: every merge of a run required ctr, prop and arena position to
// continue and kind, container and string generation to be equal, so the run's end counter (ctr + atoms), end
// position (prop + atoms), arena end (f1) and generation are those of its last row, and those are all the
// left-hand side of the test reads.  Map and tree ops never merge.  Deletes are not pairwise: after a merge a
// one-element ("bidi") span has a direction (xop_merge), so runs of delete rows are resolved serially inside the
// warp, on shuffled registers, with `back` carried across the 32-row chunks.
//
// warp per change: per-row records, XF_HEAD, the summary of the change (estimate = per merged op: List
// 4 x atoms, Text bytes, Del 8, Map 3, Tree 8, which for List / Text is the sum over its rows), segment count (XF_SEG
// marks when no op has to be cut, a synthetic-row count otherwise; the rare split paths run on lane 0).
__global__ void k_exp_changes(DocInfo* __restrict__ docs, u64 n_changes, const __grid_constant__ BatchTables t) {
    const u64 ch = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const u32 lane = threadIdx.x & 31;
    if (ch >= n_changes) return;   // (whole warps, as are the returns below)
    if (t.x_req && !t.x_req[t.blocks[t.ch_block[ch]].doc]) return;
    if (!t.ch_applied[ch]) { if (lane == 0) { t.ch_nseg[ch] = 0; t.ch_syn[ch] = 0; } return; }
    const u32 doc = t.blocks[t.ch_block[ch]].doc;
    const DocInfo& di = docs[doc];
    const u64 r0 = t.ch_op0[ch];
    const u32 nr = t.ch_nops[ch];
    // arena positions of the rows (relative to the document): a warp scan per chunk plus what the chunks before used
    u32 vals = (u32)(t.ch_aval0[ch] - t.ch_aval0[di.ch0]), strs = (u32)(t.ch_astr0[ch] - t.ch_astr0[di.ch0]);
    // a change whose head the document already had entered the store as a slice (oplog.rs:181-196): rows before the
    // cut are not part of it, the row under the cut loses its first atoms.  The counters of a change's rows increase,
    // so the rows cut away are a prefix and r_first is final before the first kept row.
    const u32 trim = t.ch_trim[ch];
    const i32 cut = t.ch_counter[ch] + (i32)trim;
    u32 r_first = 0, skip = 0;
    u32 est_ops = 0, nm = 0, ndel = 0, last_head = 0;
    bool bad = false;
    // lane 0: row r - 1 (the last row of the previous chunk) as the fields the pairwise test reads
    u32 c_xk = XK_NONE, c_cidx = 0, c_atoms = 0, c_f1 = 0, c_g = 0;
    i32 c_ctr = 0, c_prop = 0;
    bool c_del = false;   // the previous chunk's last row is a kept delete
    XOp back;             // (the same in every lane) the merged delete the last delete row ended in
    back.xk = XK_NONE;
    for (u32 c0 = 0; c0 < nr; c0 += 32) {
        const u32 r = c0 + lane;
        const bool in = r < nr;
        const u64 row = r0 + r;
        const u32 len = in ? t.op_len[row] : 0;
        const u32 ar = in ? xr_arena(t, di, row) : XA_NONE;
        const u32 nv = ar == XA_VAL ? len : 0, ns = ar == XA_STR ? t.r_bytes[row] : 0;
        const u32 iv = warp_incl_scan_u32(nv, lane), is = warp_incl_scan_u32(ns, lane);
        const u32 astart = ar == XA_STR ? strs + is - ns : (ar == XA_VAL ? vals + iv - nv : 0);
        vals += __shfl_sync(LB_FULL, iv, 31);
        strs += __shfl_sync(LB_FULL, is, 31);
        const i32 ctr = in ? t.op_counter[row] : 0;
        const bool drop = in && trim && ctr + (i32)len <= cut;
        const u32 dm = __ballot_sync(LB_FULL, drop);
        if (dm) r_first = c0 + 32 - __clz(dm);
        const bool kept = in && !drop;
        XOp o;
        o.xk = XK_NONE; o.cidx = 0; o.ctr = 0; o.atoms = 0; o.prop = 0; o.f0 = o.f1 = 0; o.f2 = 0; o.g = 0;
        o.st0 = 0; o.nst = 1;
        if (kept) {
            o = xop_resolve(t, di, (u32)ch, row, astart);
            t.x_rec[row] = xop_pack(o);
            if (o.xk == XK_NONE) bad = true;
            if (r == r_first && trim && ctr < cut) { skip = (u32)(cut - ctr); xop_slice_front(t, o, row, skip); }
        } else if (in) {
            t.x_rec[row] = mk4(0, 0, 0, 0);
            t.r_flag[row] = 0;
        }
        // row r - 1 (lane 0 takes what it kept from the previous chunk; the rotation hands it this chunk's last row)
        XOp p;
        const int src = (lane + 31) & 31;
        p.xk = (u8)__shfl_sync(LB_FULL, (u32)o.xk, src);
        p.cidx = __shfl_sync(LB_FULL, o.cidx, src);
        p.ctr = __shfl_sync(LB_FULL, o.ctr, src);
        p.atoms = __shfl_sync(LB_FULL, o.atoms, src);
        p.prop = __shfl_sync(LB_FULL, o.prop, src);
        p.f1 = __shfl_sync(LB_FULL, o.f1, src);
        p.g = __shfl_sync(LB_FULL, o.g, src);
        p.f0 = 0; p.f2 = 0; p.st0 = 0; p.nst = 1;
        if (lane == 0) {
            const u32 xk = p.xk, cidx = p.cidx, atoms = p.atoms, f1 = p.f1, g = p.g;
            const i32 pc = p.ctr, pp = p.prop;
            p.xk = (u8)c_xk; p.cidx = c_cidx; p.ctr = c_ctr; p.atoms = c_atoms; p.prop = c_prop; p.f1 = c_f1; p.g = c_g;
            c_xk = xk; c_cidx = cidx; c_ctr = pc; c_atoms = atoms; c_prop = pp; c_f1 = f1; c_g = g;
        }
        bool head = !(kept && o.xk != XK_DEL && r > r_first && xop_mergable(p, o));
        // the delete rows, in row order
        const u32 delm = __ballot_sync(LB_FULL, kept && o.xk == XK_DEL);
        for (u32 m = delm; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            XOp d;
            d.xk = XK_DEL;
            d.cidx = __shfl_sync(LB_FULL, o.cidx, j);
            d.ctr = __shfl_sync(LB_FULL, o.ctr, j);
            d.atoms = __shfl_sync(LB_FULL, o.atoms, j);
            d.prop = __shfl_sync(LB_FULL, o.prop, j);
            d.f0 = __shfl_sync(LB_FULL, o.f0, j);
            d.f1 = __shfl_sync(LB_FULL, o.f1, j);
            d.f2 = __shfl_sync(LB_FULL, o.f2, j);
            d.g = 0; d.st0 = 0; d.nst = 1;
            const bool prev_del = j ? ((delm >> (j - 1)) & 1u) != 0 : c_del;
            const bool merge = c0 + (u32)j > r_first && prev_del && xop_mergable(back, d);
            if (merge) xop_merge(back, d);
            else back = d;
            if (lane == (u32)j) head = !merge;
        }
        c_del = (delm >> 31) & 1u;
        if (kept) t.r_flag[row] = head ? XF_HEAD : 0;
        const u32 hm = __ballot_sync(LB_FULL, kept && head);
        nm += __popc(hm);
        ndel += __popc(hm & delm);
        if (hm) last_head = c0 + 31 - __clz(hm);
        const bool ins = o.xk == XK_LIST || o.xk == XK_TEXT;
        est_ops += warp_sum_u32(kept && (ins || head) ? xop_estimate(o) : 0);
    }
    bad = __any_sync(LB_FULL, bad);
    skip = warp_sum_u32(skip);   // (one lane at most)
    __syncwarp();                // the rows' flags are read by the split walk below
    if (lane) return;
    const u32 ndeps = t.ch_ndeps[ch] + (t.ch_dep_self[ch] ? 1u : 0u);
    const u32 est0 = 4 + (ndeps > 1 ? (ndeps - 1) * 4 : 0);
    u32 nseg = 1, nsyn = 0;
    t.ch_syn[ch] = 0;   // (xop_from_row below must see the decoded rows)
    if (trim && est0 + est_ops > LB_MAX_BLOCK_SIZE) {
        bad = true;   // a trimmed change that also has to be split over several blocks: not covered
        t.r_flag[r0 + (r_first < nr ? r_first : 0)] |= XF_SEG;
    } else if (est0 + est_ops > LB_MAX_BLOCK_SIZE) {
        XSplit sp = split_change(t, di, (u32)ch, r0, nr, est0, [&](u64 row, u32 a, u32, bool, bool seg) {
            if (seg && a == 0) t.r_flag[row] |= XF_SEG;   // valid when nothing gets cut (else the synthetic rows carry it)
        });
        nseg = sp.nseg;
        if (sp.sliced && nseg > 1) nsyn = sp.nsyn;   // (a lone "slice" that is the whole op changes nothing)
    } else t.r_flag[r0 + (r_first < nr ? r_first : 0)] |= XF_SEG;
    t.ch_nseg[ch] = nseg;
    t.ch_novf[ch] = nseg - 1;
    t.ch_syn[ch] = nsyn;
    if (nseg == 1) {   // the common case: the change is its own (only) segment, summarised right here
        t.sg_src[ch] = (u32)ch; t.sg_r0[ch] = r_first; t.sg_from[ch] = trim; t.sg_atoms[ch] = t.ch_len[ch] - trim; t.sg_est[ch] = est_ops;
        t.sg_nmops[ch] = nm; t.sg_ndel[ch] = ndel; t.sg_nrows[ch] = nr - r_first; t.sg_last_head[ch] = last_head; t.sg_skip[ch] = skip;
    }
    if (bad) atomicOr(&t.xdoc[doc].flags, 1u);
}

// thread per change, the changes k_exp_changes found to span several segments: synthetic rows, summaries
__global__ void k_exp_split_changes(DocInfo* __restrict__ docs, u64 n_changes, const __grid_constant__ BatchTables t) {
    u64 ch = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_changes) return;
    if (t.x_req && !t.x_req[t.blocks[t.ch_block[ch]].doc]) return;
    if (!t.ch_applied[ch] || t.ch_nseg[ch] <= 1) return;
    const DocInfo& di = docs[t.blocks[t.ch_block[ch]].doc];
    u64 r0 = t.ch_op0[ch];
    u32 nr = t.ch_nops[ch];
    u32 ndeps = t.ch_ndeps[ch] + (t.ch_dep_self[ch] ? 1u : 0u);
    u32 est0 = 4 + (ndeps > 1 ? (ndeps - 1) * 4 : 0);
    u32 nsyn = t.ch_syn[ch];
    if (nsyn) {
        // materialise the synthetic rows: a copy of every untouched row, one row per slice of a cut insert
        u64 s0 = t.ch_syn0[ch];
        u32 w = 0;
        t.ch_syn[ch] = 0;   // the walk reads the decoded rows
        split_change(t, di, (u32)ch, r0, nr, est0, [&](u64 row, u32 a, u32 b, bool head, bool seg) {
            u64 i = s0 + w++;
            uint4 rec = t.x_rec[row];
            u32 xk = rec.x & 7u;
            u32 ra = t.op_len[row];
            const u8* pp; u32 pn;
            xr_payload(t, row, xk, &pp, &pn);
            u32 b0 = 0, b1 = pn;
            if (xk == XK_TEXT) { b0 = text_byte_index(pp, pn, ra, a); b1 = text_byte_index(pp, pn, ra, b); }
            else if (xk == XK_LIST && (a != 0 || b != ra)) {   // byte span of items [a,b)
                Cur c(pp, pn);
                for (u32 k = 0; k < a && !c.err; k++) { u8 kk = c.get(); skip_loro_value_content(c, kk, nullptr); }
                b0 = (u32)(c.p - pp);
                for (u32 k = a; k < b && !c.err; k++) { u8 kk = c.get(); skip_loro_value_content(c, kk, nullptr); }
                b1 = (u32)(c.p - pp);
            }
            if (xk == XK_LIST || xk == XK_TEXT) {
                rec.y += a;                                   // counter
                rec.z += a;                                   // position
                rec.w += xk == XK_TEXT ? b0 : a;              // arena start
            }
            t.s_rec[i] = rec;
            t.s_len[i] = b - a;
            t.s_bytes[i] = xk == XK_TEXT ? b1 - b0 : 0;
            t.s_voff[i] = (u64)(pp - t.bytes) + b0;
            t.s_vlen[i] = b1 - b0;
            t.s_aux[i] = xk == XK_TEXT ? str_gen(t.x_rec[row].w + t.r_bytes[row]) : t.op_aux[row];
            t.s_flag[i] = (head ? XF_HEAD : 0) | (seg ? XF_SEG : 0);
        });
        t.ch_syn[ch] = nsyn;
    }
    segment_summaries(t, di, (u32)ch);
}

// ---------------------------------------------------------------------------------------------- B + C: the stores
struct XEntry {        // a change on its way through a store: one segment, or a run of merged ones
    u32 src, from;     // metadata of its first segment: source change + atom offset (deps, lamport, timestamp, message)
    u32 pos, r0;       // where its rows start: position in ch_aorder (absolute) + row inside that change
    u32 atoms, est_ops, nmops, ndel, nrows;
    u32 skip;          // atoms of the first row outside the entry (import-side trim, or the front cut of its span)
    u32 tail;          // atoms of the last row outside the entry (the end cut of its span)
    u32 lh_ch, lh_row; // last op: source change + row (inside that change) of its first row ...
    XOp last;          // ... or, once the entry has been through a store, the accumulated op itself
    bool last_valid;
};
struct XStore {
    bool have_block, open_valid, open_starts_block;
    u32 blk_est;
    XEntry open;       // the store's last change (still able to absorb the next one)
    XOp back;          // last op of `open`, accumulated
};
__device__ __forceinline__ bool xmsg_same(const BatchTables& t, u32 a, u32 b) {
    u32 la = t.ch_msg_len[a], lb = t.ch_msg_len[b];
    if (la != lb) return false;
    const u8* pa = t.bytes + t.ch_msg_off[a];
    const u8* pb = t.bytes + t.ch_msg_off[b];
    for (u32 i = 0; i < la; i++)
        if (pa[i] != pb[i]) return false;
    return true;
}
__device__ __forceinline__ u32 xentry_ndeps(const BatchTables& t, const XEntry& e) {
    return e.from ? 1u : t.ch_ndeps[e.src] + (t.ch_dep_self[e.src] ? 1u : 0u);
}
// cursor over the rows of an entry in store order (rows of consecutive applied changes of the peer)
struct XRows {
    const BatchTables& t; u32 pos; u32 r; u32 ch; u32 nr; u64 row0;
    u32 skip;   // atoms of the CURRENT row that are not part of the store (first kept row of a trimmed change); the
                // creator of the cursor knows the skip of the row it starts on (entry / final-change records)
    __device__ XRows(const BatchTables& t_, u32 pos_, u32 r_) : t(t_), pos(pos_), r(r_), skip(0) { load(); }
    __device__ void load() { ch = t.ch_aorder[pos]; change_rows(t, ch, &row0, &nr); }
    __device__ u64 row() const { return row0 + r; }
    __device__ void next() {
        r++;
        skip = 0;
        while (r >= nr) {
            pos++; r = 0; ch = t.ch_aorder[pos];
            if (!t.ch_applied[ch]) { nr = 0; continue; }
            change_rows(t, ch, &row0, &nr);
            if (t.ch_trim[ch]) { r = t.sg_r0[ch]; skip = t.sg_skip[ch]; }   // a trimmed change starts at its first kept row
        }
    }
};
// accumulate the merged op that starts at the cursor (consumes its rows, at most `left` of them): `skip` atoms of its
// first row are left out, and `tail` atoms of the entry's last row when the op reaches it (the cursor then stays there)
__device__ inline XOp xop_gather(const BatchTables& t, const DocInfo& di, XRows& it, u32& left, u32 skip = 0, u32 tail = 0) {
    XOp o = xop_from_row(t, di, it.ch, it.row());
    if (skip) xop_slice_front(t, o, it.row(), skip);
    left--;
    if (left) it.next();
    while (left && !(xr_flag(t, it.row()) & XF_HEAD)) {
        XOp x = xop_from_row(t, di, it.ch, it.row());
        if (it.skip) xop_slice_front(t, x, it.row(), it.skip);
        xop_merge(o, x);
        left--;
        if (left) it.next();
    }
    if (!left && tail) xop_slice_back(t, o, it.row(), tail);
    return o;
}
// last op of an entry that came straight from stage A: from its head row to the end of its segment
__device__ inline XOp xentry_last_op(const BatchTables& t, const DocInfo& di, const XEntry& E) {
    if (E.last_valid) return E.last;
    u64 row0;
    u32 nr;
    change_rows(t, E.lh_ch, &row0, &nr);
    XOp o = xop_from_row(t, di, E.lh_ch, row0 + E.lh_row);
    if (E.skip && E.lh_row == E.r0 && E.lh_ch == t.ch_aorder[E.pos]) xop_slice_front(t, o, row0 + E.lh_row, E.skip);
    u32 r = E.lh_row + 1;
    while (r < nr && !(xr_flag(t, row0 + r) & (XF_HEAD | XF_SEG))) { xop_merge(o, xop_from_row(t, di, E.lh_ch, row0 + r)); r++; }
    return o;
}
// ChangeStore::insert_change + ChangesBlock::push_change (change_store.rs:711-764, 1244-1291): E is the next change
// of the peer.  Returns true when the store's previous last change is complete (copied to `done`).
__device__ inline bool xstore_push(const BatchTables& t, const DocInfo& di, XStore& s, const XEntry& E, XEntry& done,
                                   bool& done_starts_block) {
    u32 nd = xentry_ndeps(t, E);
    u32 est = 4 + E.est_ops + (nd > 1 ? (nd - 1) * 4 : 0);
    bool new_block = true;
    if (s.have_block) {
        bool is_full = est + s.blk_est > LB_MAX_BLOCK_SIZE;
        bool dep_only_self = E.from ? true : (t.ch_dep_self[E.src] && t.ch_ndeps[E.src] == 0);
        bool can = dep_only_self && t.ch_ts[E.src] <= t.ch_ts[s.open.src] && xmsg_same(t, s.open.src, E.src);
        // the last change ends inside a row (an end cut) and E starts on that row: E can only grow the change when the
        // two halves of the row's op merge back (for list, text and delete halves they always do), since the grown
        // change lists the row once; otherwise E starts a change of its own
        const bool shared = s.open.tail != 0;
        if (can && shared) {
            XRows it(t, E.pos, E.r0);
            u32 left = E.nrows;
            can = xop_mergable(s.back, xop_gather(t, di, it, left, E.skip, E.tail));
        }
        bool single = false;
        if (can && is_full && E.nmops == 1) {
            XRows it(t, E.pos, E.r0);
            u32 left = E.nrows;
            single = xop_mergable(s.back, xop_gather(t, di, it, left, E.skip, E.tail));
        }
        if (can && (!is_full || single)) {
            // the ops of E are pushed onto the last change (RleVec::push): a prefix of them may merge into its last op.
            // When the last change ends inside a row (an end cut), E starts on that same row: the two halves of the row's
            // op merge back, and the grown change lists the row once
            XRows it(t, E.pos, E.r0);
            u32 left = E.nrows;
            u32 merged = 0, merged_sz = 0, merged_del = 0;
            bool first_op = true;
            while (left) {
                u64 head_row = it.row();
                XOp o = xop_gather(t, di, it, left, first_op ? E.skip : it.skip, E.tail);
                if (!xop_mergable(s.back, o)) break;
                merged_sz += xop_estimate(o);
                merged_del += o.xk == XK_DEL;
                xop_merge(s.back, o);
                if (!(first_op && shared)) *xr_flagp(t, head_row) &= (u8)~XF_HEAD;
                first_op = false;
                merged++;
            }
            s.blk_est += E.est_ops - merged_sz;          // only ops that did not merge count (change_store.rs:1271-1279)
            s.open.atoms += E.atoms;
            s.open.est_ops += E.est_ops - 8 * merged_del; // fresh estimate of the grown change (used by the next store)
            s.open.nmops += E.nmops - merged;
            s.open.ndel += E.ndel - merged_del;
            s.open.nrows += E.nrows - (shared ? 1u : 0u);
            s.open.tail = E.tail;
            if (E.nmops > merged) s.back = xentry_last_op(t, di, E);
            return false;
        }
        if (!is_full) { s.blk_est += est; new_block = false; }
    }
    bool closed = s.open_valid;
    if (closed) { done = s.open; done.last = s.back; done.last_valid = true; done_starts_block = s.open_starts_block; }
    if (new_block) { s.have_block = true; s.blk_est = est; }
    s.open = E;
    s.open_valid = true;
    s.open_starts_block = new_block;
    s.back = xentry_last_op(t, di, E);
    return closed;
}

// Change::slice (change_store.rs:505-521, change.rs:203-258) in front: entry E covers counters [c0, c0 + atoms) of its
// peer; its first `cut` atoms (0 < cut < atoms) are dropped.  The summary is left to xentry_summary.
__device__ inline void xentry_trim_front(const BatchTables& t, XEntry& E, u32 cut) {
    XRows it(t, E.pos, E.r0);
    u32 left = E.nrows, acc = 0, lead = E.skip;   // `lead`: atoms of the current row already outside the entry
    while (left) {
        u32 len = xr_len(t, it.row()) - lead;
        if (acc + len > cut) break;
        acc += len;
        left--;
        if (left) { it.next(); lead = it.skip; } else lead = 0;
    }
    E.pos = it.pos;
    E.r0 = it.r;
    E.nrows = left;
    E.skip = lead + (cut - acc);
    E.from += cut;
    E.atoms -= cut;
}
// ... and at the end: only the first `keep` atoms (0 < keep < atoms) stay; the row holding the last of them ends the
// entry, with the atoms after it counted in `tail` (E.tail is 0 before: end cuts are taken from the import store)
__device__ inline void xentry_trim_back(const BatchTables& t, XEntry& E, u32 keep) {
    XRows it(t, E.pos, E.r0);
    u32 n = 1, acc = 0, lead = E.skip;
    while (true) {
        const u32 len = xr_len(t, it.row()) - lead;
        if (acc + len >= keep) { E.tail = acc + len - keep; break; }
        acc += len;
        n++;
        it.next();
        lead = it.skip;
    }
    E.nrows = n;
    E.atoms = keep;
}
// fresh summary of a cut entry: size estimate, ops, deletes, last op
__device__ inline void xentry_summary(const BatchTables& t, const DocInfo& di, XEntry& E) {
    XRows it(t, E.pos, E.r0);
    u32 l = E.nrows, est = 0, nm = 0, nd = 0;
    XOp last;
    last.xk = XK_NONE;
    bool first = true;
    while (l) {
        XOp o = xop_gather(t, di, it, l, first ? E.skip : it.skip, E.tail);
        first = false;
        est += xop_estimate(o);
        nm++;
        nd += o.xk == XK_DEL;
        last = o;
    }
    E.est_ops = est;
    E.nmops = nm;
    E.ndel = nd;
    E.last = last;
    E.last_valid = true;
}
// Change::slice(start, end) clamped to the entry, which overlaps [start, end).  The summary is left to xentry_summary.
__device__ inline void xentry_slice(const BatchTables& t, XEntry& E, i32 start, i32 end) {
    const i32 c0 = t.ch_counter[E.src] + (i32)E.from;
    if (start > c0) xentry_trim_front(t, E, (u32)(start - c0));
    const i32 c1 = t.ch_counter[E.src] + (i32)E.from;
    if (end < c1 + (i32)E.atoms) xentry_trim_back(t, E, (u32)(end - c1));
}

// The import store of one peer, rebuilt from its segments in counter order through xstore_push (insert_change merges,
// MAX_BLOCK_SIZE splits, RleVec op merges written to the rows' XF_HEAD flags).  Every change the store completes goes to
// take(change), and at the end its open change, with its accumulated last op.  more() is asked before each change of
// the peer and before that last one: once it is false, the walk stops.
template <class More, class Take>
__device__ inline void xstore_walk(const BatchTables& t, const DocInfo& di, const DocPeer& dp, More more, Take take) {
    XStore s1;
    s1.have_block = s1.open_valid = s1.open_starts_block = false; s1.blk_est = 0;
    XEntry done;
    bool done_blk = false;
    for (u32 k = 0; k < dp.ch_count && more(); k++) {
        u32 pos = (u32)di.ch0 + dp.ch_first + k;
        u32 ch = t.ch_aorder[pos];
        u32 nseg = t.ch_nseg[ch];
        for (u32 q = 0; q < nseg; q++) {
            u64 sg = q == 0 ? (u64)ch : t.n_changes + t.ch_seg0[ch] + q - 1;
            XEntry E;
            E.src = ch; E.from = t.sg_from[sg]; E.pos = pos; E.r0 = t.sg_r0[sg]; E.atoms = t.sg_atoms[sg];
            E.est_ops = t.sg_est[sg]; E.nmops = t.sg_nmops[sg]; E.ndel = t.sg_ndel[sg]; E.nrows = t.sg_nrows[sg];
            E.lh_ch = ch; E.lh_row = t.sg_last_head[sg]; E.last_valid = false; E.skip = t.sg_skip[sg]; E.tail = 0;
            if (xstore_push(t, di, s1, E, done, done_blk)) take(done);
        }
    }
    if (s1.open_valid && more()) {
        s1.open.last = s1.back;
        s1.open.last_valid = true;
        take(s1.open);
    }
}

// first final-change slot of a document: one slot per segment, and in an export of chosen spans one more per span of
// the documents before it (a stored change that k spans cut leaves k pieces, so a document can need that many more)
__device__ __forceinline__ u64 xfc0(const BatchTables& t, const DocInfo& di) {
    return di.ch0 + t.ch_seg0[di.ch0] + (t.x_span0 ? t.x_span0[di.peer0] : 0u);
}
// thread per document: per peer, the import store (s1) is rebuilt once; every change it completes is cut to each of the
// peer's spans it overlaps (one change can give several pieces, each cut at both ends) and the pieces enter the export
// store (s2) in counter order.  A span with the fresh bit starts a new block there (its first change found no block of
// the peer ending at its start: change_store.rs:711-764); the others continue the block of the span that ends at their
// start.
__global__ void k_exp_store(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK) return;
    XDoc x = t.xdoc[d];
    if (t.x_req && !t.x_req[d]) { x.n_fc = x.n_mb = 0; t.xdoc[d] = x; return; }
    if (x.flags & 1) { t.xdoc[d] = x; return; }
    u64 w = xfc0(t, di);
    u64 w0 = w;
    u32 n_mb = 0;
    auto emit = [&](const XEntry& e, bool starts_block) {
        t.fc_src[w] = e.src; t.fc_pos[w] = e.pos; t.fc_r0[w] = e.r0; t.fc_from[w] = e.from; t.fc_atoms[w] = e.atoms;
        t.fc_nrows[w] = e.nrows; t.fc_ndel[w] = e.ndel; t.fc_block[w] = starts_block ? 1 : 0; t.fc_skip[w] = e.skip;
        t.fc_tail[w] = e.tail; t.fc_est[w] = e.est_ops;
        n_mb += starts_block;
        w++;
    };
    for (u32 rank = 0; rank < di.P; rank++) {   // blocks are keyed by (peer id, counter): ascending peer id
        u32 p = 0;
        while (p < di.P && t.dpeer[di.peer0 + p].rank != rank) p++;
        if (p == di.P) break;
        const DocPeer& dp = t.dpeer[di.peer0 + p];
        const u32 sp0 = t.x_spans ? t.x_span0[di.peer0 + p] : 0u;
        const u32 nsp = t.x_spans ? t.x_span0[di.peer0 + p + 1] - sp0 : 1u;
        u32 j = 0;   // the first span not yet finished
        XStore s2;   // export store
        s2.have_block = s2.open_valid = s2.open_starts_block = false; s2.blk_est = 0;
        // each change of the import store: its pieces inside the spans go to the export store; the walk ends with the spans
        xstore_walk(t, di, dp, [&] { return j < nsp; }, [&](const XEntry& c) {
            const i32 c0 = t.ch_counter[c.src] + (i32)c.from, c1 = c0 + (i32)c.atoms;
            while (j < nsp) {
                XSpan s;
                if (t.x_spans) s = t.x_spans[sp0 + j];
                else { s.start = 0; s.end = dp.end_counter; s.fresh = 1; }
                if (s.start >= c1) break;
                if (s.end > c0) {
                    if (s.fresh && s.start >= c0) {
                        if (s2.open_valid) emit(s2.open, s2.open_starts_block);
                        s2.have_block = s2.open_valid = false;
                    }
                    XEntry piece = c;
                    if (s.start > c0 || s.end < c1) {
                        xentry_slice(t, piece, s.start, s.end);
                        xentry_summary(t, di, piece);
                    }
                    XEntry d2;
                    bool d2_blk = false;
                    if (xstore_push(t, di, s2, piece, d2, d2_blk)) emit(d2, d2_blk);
                }
                if (s.end > c1) break;
                j++;
            }
        });
        if (s2.open_valid) emit(s2.open, s2.open_starts_block);
    }
    x.n_fc = (u32)(w - w0);
    x.n_mb = n_mb;
    t.xdoc[d] = x;
}

// Staging slot of an output block, in bytes: the store's size estimate of its changes (text bytes, 4 per list item,
// 8 per delete span, 3 per map op) plus room for the op and delete columns, the per-change metadata and the
// registers.  This is what the blocks usually need, not a bound (a bound is about 40 bytes per row against about 8
// used): the few blocks that outgrow their slot are encoded again, into a slot of their exact size (k_exp_layout).
__device__ __forceinline__ u64 xstage_change(const BatchTables& t, u64 k) {
    return t.fc_est[k] + 4ull * t.fc_nrows[k] + 4ull * t.fc_ndel[k] + 16;
}
__device__ __forceinline__ u64 xstage_block(const DocInfo& di) { return 64 + 8ull * (di.P + di.C); }
// Scratch words of an output block, as the encoder carves them: the peer, key and container registers (order and
// inverse each), then four op columns per row (five in documents with tree ops: the position ranks) and three delete
// columns per delete.
__device__ __forceinline__ u64 xscratch_change(const BatchTables& t, const XDoc& x, u64 k) {
    return (4ull + ((x.flags >> 1) & 1u)) * t.fc_nrows[k] + 3ull * t.fc_ndel[k];
}
__device__ __forceinline__ u64 xscratch_block(const DocInfo& di) { return 2ull * (di.P + di.K + di.C); }

// thread per document: list the output blocks (after the scans of n_mb, scratch and staging sizes).  stage_max caps
// every slot's capacity (testing: sends the blocks that need more through the retry)
__global__ void k_exp_list(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t, XBlock* __restrict__ xb, u32 stage_max) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    const XDoc& x = t.xdoc[d];
    if (di.code != DOC_OK || x.n_mb == 0) return;
    u64 f0 = xfc0(t, di);
    u64 scr = x.scratch0, stg = x.stage0, words = 0, slot = 0;
    int idx = -1;
    XBlock b;
    memset(&b, 0, sizeof(b));
    auto close = [&]() {
        b.stage_cap = (u32)(slot < stage_max ? slot : stage_max);
        xb[x.ob0 + idx] = b;
        scr += words;
        stg += slot;
    };
    for (u64 k = f0; k < f0 + x.n_fc; k++) {
        if (t.fc_block[k]) {
            if (idx >= 0) { b.fc1 = (u32)k; close(); }
            idx++;
            memset(&b, 0, sizeof(b));
            b.doc = d; b.fc0 = (u32)k; b.scratch = scr; b.stage = stg;
            words = xscratch_block(di);
            slot = xstage_block(di);
        }
        b.n_rows += t.fc_nrows[k];
        b.n_dels += t.fc_ndel[k];
        words += xscratch_change(t, x, k);
        slot += xstage_change(t, k);
    }
    if (idx >= 0) { b.fc1 = (u32)(f0 + x.n_fc); close(); }
}
// thread per document: scratch words and staging bytes of its blocks
__global__ void k_exp_sizes(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t, u32* __restrict__ n_blocks,
                            u32* __restrict__ n_scratch, u32* __restrict__ n_stage) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    const XDoc& x = t.xdoc[d];
    u32 nb = di.code == DOC_OK ? x.n_mb : 0;
    u64 words = 0, bytes = 0;
    if (nb) {
        u64 f0 = xfc0(t, di);
        words = nb * xscratch_block(di);
        bytes = nb * xstage_block(di);
        for (u64 k = f0; k < f0 + x.n_fc; k++) {
            words += xscratch_change(t, x, k);
            bytes += xstage_change(t, k);
        }
    }
    n_blocks[d] = nb;
    n_scratch[d] = (u32)words;
    n_stage[d] = (u32)bytes;
}

// ---------------------------------------------------------------------------------------------- column encoders
// All work on an index range with a value functor, so that a literal segment's length is known before its values
// are written (serde_columnar AnyRle state machine: maximal runs of >= 2 equal values become runs, the values
// between them literal segments; a lone value is a literal of one).
// The values come out of per-block scratch columns in global memory and every scan below is a chain of dependent
// loads: the scans fetch four values at a time -- the loads are independent of each other and of the comparisons --
// and consume them in order.
template <class F, class W>
__device__ inline void enc_anyrle(XSink& s, u32 n, F val, W wr) {
    u32 i = 0;
    while (i < n) {
        i64 v = val(i);
        u32 j = i;
        while (j + 1 < n) {
            const u32 base = j + 1, m = n - base < 4 ? n - base : 4;
            i64 w0 = val(base), w1 = m > 1 ? val(base + 1) : 0, w2 = m > 2 ? val(base + 2) : 0, w3 = m > 3 ? val(base + 3) : 0;
            u32 q = 0;
            if (w0 == v) { q = 1; if (m > 1 && w1 == v) { q = 2; if (m > 2 && w2 == v) { q = 3; if (m > 3 && w3 == v) q = 4; } } }
            j += q;
            if (q < m) break;
        }
        if (j > i) {
            s.zigzag((i64)(j - i + 1));
            wr(s, v);
            i = j + 1;
            continue;
        }
        u32 k = i;
        i64 cur = v;
        while (k < n) {
            const u32 base = k + 1;
            if (base >= n) { k++; break; }
            const u32 m = n - base < 4 ? n - base : 4;
            i64 w[4];
            w[0] = val(base); w[1] = m > 1 ? val(base + 1) : 0; w[2] = m > 2 ? val(base + 2) : 0; w[3] = m > 3 ? val(base + 3) : 0;
            bool stop = false;
#pragma unroll
            for (u32 q = 0; q < 4; q++) {
                if (q >= m || stop) break;
                if (w[q] == cur) { stop = true; break; }
                cur = w[q];
                k++;
            }
            if (stop) break;
        }
        s.zigzag(-(i64)(k - i));
        {
            u32 q = i;
            for (; q + 4 <= k; q += 4) {
                i64 a = val(q), b = val(q + 1), c = val(q + 2), d = val(q + 3);
                wr(s, a); wr(s, b); wr(s, c); wr(s, d);
            }
            for (; q < k; q++) wr(s, val(q));
        }
        i = k;
    }
}
struct WrVarint { __device__ void operator()(XSink& s, i64 v) const { s.varint((u64)v); } };
struct WrByte { __device__ void operator()(XSink& s, i64 v) const { s.put((u8)v); } };
struct WrZigzag { __device__ void operator()(XSink& s, i64 v) const { s.zigzag(v); } };
template <class F>
__device__ inline void enc_deltarle(XSink& s, u32 n, F val) {   // AnyRle over the deltas from 0
    enc_anyrle(s, n, [&](u32 i) -> i64 { i64 prev = i ? val(i - 1) : 0; return val(i) - prev; }, WrZigzag());
}
template <class F>
__device__ inline void enc_boolrle(XSink& s, u32 n, F val) {
    if (n == 0) return;
    bool state = false;
    u64 run = 0;
    for (u32 i = 0; i < n; i++) {
        bool b = val(i);
        if (b == state) run++;
        else { s.varint(run); state = !state; run = 1; }
    }
    s.varint(run);
}
struct XBits {   // MSB-first bit packer on top of a sink
    XSink& s;
    u32 cur;
    int nbits;
    __device__ XBits(XSink& s_) : s(s_), cur(0), nbits(0) {}
    __device__ void bit(bool b) {
        cur = (cur << 1) | (b ? 1u : 0u);
        if (++nbits == 8) { s.put((u8)cur); cur = 0; nbits = 0; }
    }
    __device__ void bits(u64 v, int n) { for (int i = n - 1; i >= 0; i--) bit((v >> i) & 1); }
};
// DeltaOfDelta (docs/encoding.md:1126-1172): Option<i64> first, u8 bits used in the last byte, prefix codes
template <class F>
__device__ inline void enc_dod(XSink& s, u32 n, F val) {
    if (n == 0) { s.put(0); s.put(0); return; }
    s.put(1);
    s.zigzag(val(0));
    if (n == 1) { s.put(0); return; }
    // the "bits used" byte precedes the packed bits: count them first
    u64 total_bits = 0;
    {
        i64 prev_delta = 0;
        for (u32 i = 1; i < n; i++) {
            i64 dl = val(i) - val(i - 1);
            i64 x = dl - prev_delta;
            prev_delta = dl;
            if (x == 0) total_bits += 1;
            else if (x >= -63 && x <= 64) total_bits += 9;
            else if (x >= -255 && x <= 256) total_bits += 12;
            else if (x >= -2047 && x <= 2048) total_bits += 16;
            else if (x >= -1048575 && x <= 1048576) total_bits += 26;
            else total_bits += 69;
        }
    }
    int used = (int)(total_bits & 7);
    s.put((u8)(used == 0 ? 8 : used));
    XBits bw(s);
    i64 prev_delta = 0;
    for (u32 i = 1; i < n; i++) {
        i64 dl = val(i) - val(i - 1);
        i64 x = dl - prev_delta;
        prev_delta = dl;
        if (x == 0) bw.bit(false);
        else if (x >= -63 && x <= 64) { bw.bits(2, 2); bw.bits((u64)(x + 63), 7); }
        else if (x >= -255 && x <= 256) { bw.bits(6, 3); bw.bits((u64)(x + 255), 9); }
        else if (x >= -2047 && x <= 2048) { bw.bits(14, 4); bw.bits((u64)(x + 2047), 12); }
        else if (x >= -1048575 && x <= 1048576) { bw.bits(30, 5); bw.bits((u64)(x + 1048575), 21); }
        else { bw.bits(31, 5); bw.bits((u64)x, 64); }
    }
    if (bw.nbits) s.put((u8)((bw.cur & 0xFF) << (8 - bw.nbits)));
}

// ---------------------------------------------------------------------------------------------- encode
// First-use registers of one block (encoding/value_register.rs): order lists + inverse maps in scratch.
struct XReg {
    u32* ord; u32* inv; u32 n;
    __device__ u32 reg(u32 v) {
        if (inv[v] != 0xFFFFFFFFu) return inv[v];
        inv[v] = n;
        ord[n] = v;
        return n++;
    }
};
// LoroValues [p, p + n) copied into `s` with the key indices of nested maps translated from the source block's key
// arena (doc-level key = key_map[src_key0 + idx]) to the output block's register (write_loro_value registers a map's
// keys as it meets them: encoding/value.rs:1027-1036).
// The stack holds LB_MAX_NESTING levels, as deep as the decoder admits a value: it never fills, so a value is always
// copied whole.
__device__ inline void xvalue_copy(XSink& s, const u8* p, u32 n, const BatchTables& t, u64 src_key0, XReg& keys) {
    Cur c(p, n);
    u32 stack[LB_MAX_NESTING];
    int sp = 0;
    while (!c.err) {
        while (sp > 0 && (stack[sp - 1] & 0x7fffffffu) == 0) sp--;
        if (sp == 0 && c.empty()) return;
        if (sp > 0) {
            stack[sp - 1]--;
            if (stack[sp - 1] & 0x80000000u) {
                u32 dk = t.key_map[src_key0 + (u32)c.varint()];
                s.varint(keys.reg(dk));
            }
        }
        u8 kind = c.get();
        s.put(kind);
        switch (kind) {
            case 0: case 1: case 2: break;
            case 3: { const u8* a = c.p; (void)c.sleb(); s.copy(a, (u64)(c.p - a)); break; }
            case 4: { const u8* a = c.p; c.skip(8); s.copy(a, (u64)(c.p - a)); break; }
            case 5: case 6: { const u8* a = c.p; u64 l = c.varint(); c.skip(l); s.copy(a, (u64)(c.p - a)); break; }
            case 7: case 8: {
                u64 cnt = c.varint();
                s.varint(cnt);
                if (sp >= LB_MAX_NESTING || cnt > (1u << 28)) return;
                stack[sp++] = (u32)cnt | (kind == 8 ? 0x80000000u : 0u);
                break;
            }
            case 9: s.put(c.get()); break;
            default: return;
        }
    }
}
// cross-peer deps of the block's changes as one flat sequence (cursor: accesses are almost monotonic)
struct XDeps {
    const BatchTables& t; u32 fc0, N; u32 j; u32 base;
    __device__ XDeps(const BatchTables& t_, u32 fc0_, u32 N_) : t(t_), fc0(fc0_), N(N_), j(0), base(0) {}
    __device__ u32 nd(u32 jj) const { return t.fc_from[fc0 + jj] ? 0u : t.ch_ndeps[t.fc_src[fc0 + jj]]; }
    __device__ u64 at(u32 i) {   // index of flat dep i in the dep tables
        if (i < base) { j = 0; base = 0; }
        while (j < N) {
            u32 n = nd(j);
            if (i < base + n) return t.ch_dep0[t.fc_src[fc0 + j]] + (i - base);
            base += n;
            j++;
        }
        return 0;
    }
};
__device__ __forceinline__ u8 xk_value_type(u8 xk) {
    switch (xk) {
        case XK_LIST: case XK_MAPSET: return VK_LORO_VALUE;
        case XK_TEXT: return VK_STR;
        case XK_DEL: return VK_DELETE_SEQ;
        case XK_TREE: return VK_RAW_TREE_MOVE;
        default: return VK_DELETE_ONCE;
    }
}

// ---------------------------------------------------------------------------------------------- fractional indexes
// encode_block pre-fills its position register with the block's positions in sorted order (block_encode.rs:156-178).
// The byte-string sort happens once per document: a warp sorts the document's position entries (first eight bytes as
// the key, full comparison on ties) and hands every entry the dense rank of its bytes; a block then only sorts ranks.
__device__ inline int xpos_cmp(const BatchTables& t, u32 a, u32 b) {
    if (a == b) return 0;
    const u8* pa = t.pos_pool + t.pos_off[a];
    const u8* pb = t.pos_pool + t.pos_off[b];
    u32 la = t.pos_len[a], lb = t.pos_len[b];
    u32 n = la < lb ? la : lb;
    for (u32 i = 0; i < n; i++)
        if (pa[i] != pb[i]) return pa[i] < pb[i] ? -1 : 1;
    return la < lb ? -1 : (la > lb ? 1 : 0);
}
__global__ void k_exp_posrank(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t) {
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK || !di.has_tree) return;
    const u64 p_lo = t.blocks[di.b0].pos0;
    const u32 n = (u32)(t.blocks[di.b1].pos0 - p_lo);
    u64* key = t.ps_key + p_lo;
    u32* val = t.ps_val + p_lo;
    for (u32 i = lane; i < n; i += 32) {
        const u8* pb = t.pos_pool + t.pos_off[p_lo + i];
        u32 pl = t.pos_len[p_lo + i];
        u64 k = 0;
        for (u32 q = 0; q < 8; q++) k = (k << 8) | (q < pl ? pb[q] : 0u);
        if (k == ~0ull) k--;          // keep +inf free (the sort treats it as padding); ties fall back to the bytes
        key[i] = k;
        val[i] = i;
    }
    __syncwarp();
    warp_sort_pairs(key, val, n, lane, [&](u32 a, u32 b) -> bool { return xpos_cmp(t, (u32)p_lo + a, (u32)p_lo + b) < 0; });
    // dense ranks: a new rank starts wherever the bytes differ from the predecessor's
    u32 carry = 0;
    for (u32 j0 = 0; j0 < n; j0 += 32) {
        u32 j = j0 + (u32)lane;
        int fresh = 0;
        if (j < n) fresh = (j == 0 || xpos_cmp(t, (u32)p_lo + val[j - 1], (u32)p_lo + val[j]) != 0) ? 1 : 0;
        int incl = warp_incl_scan(fresh, lane);
        if (j < n) {
            u32 rank = carry + (u32)incl - 1;
            t.pos_rank[p_lo + val[j]] = rank;
            if (fresh) t.pos_rep[p_lo + rank] = (u32)p_lo + val[j];
        }
        carry += (u32)__shfl_sync(LB_FULL, incl, 31);
    }
    if (lane == 0) t.xdoc[d].n_prank = carry;
}

// thread per output block: gather ops into scratch columns and registers while writing the values section into the
// block's staging slot (`out` = the staging buffer), then every other section (column) writer stores its body after it
// and its length into the XBlock.  A block whose pieces outgrow the slot only counts from there on, so its lengths are
// exact, and is flagged (XBlock::ovf).  retry = 1, flagged blocks only: the same encode once more, into the slot
// k_exp_layout gave the block in the retry buffer (`out`, from the document's restage0 on), which its lengths fill.
// Two builds of the same code: <1> is compiled with __launch_bounds__(64, 5) (the compiler then schedules for 64-thread
// CTAs: 132 registers against 128 without bounds, other load / store placement), <0> without bounds.  Each has a twin,
// k_exp_encode_cut<CAPPED>, that also honours end cuts (fc_tail: an export of spans that end inside a change); the
// end-cut code costs the encoder registers (sm_90a: 136 against 128 unbounded, 136 against 132 bounded), which would
// take the unbounded build from 8 CTAs to 7, so the exports without end cuts (import time, updates(from)) keep builds
// without it.  Registers decide
// the CTAs an SM holds: up to 128 give 8, up to 136 give 7, and each build is faster at its own count.  On one H100
// 80GB HBM3 (700 W power limit), the bounded build at 127 registers (8 CTAs) took C5's re-export from 107 to 120 ms,
// and the unbounded one at 132 (7 CTAs) took C3's at 4 k documents from 38.6 to 45.9 ms.
// The host picks by the number of output blocks.  Re-export phase on one H100 80GB HBM3 (400 W power limit), unbounded
// against bounded: C3 at 4 k documents (~55 k blocks) 39.1 against 46.6 ms; C5 at 10 k documents (160 k blocks) 128.5
// against 106.4 ms; C3 at 40 k documents (~550 k blocks) 346.4 against 325.3 / 323.4 ms.  So batches of at least
// LB_XENC_BOUNDED_MIN_BLOCKS output blocks take the bounded build.
#define LB_XENC_BOUNDED_MIN_BLOCKS 100000ull
template <int CUT>
__device__ __forceinline__ void exp_encode_body(
    const DocInfo* __restrict__ docs, u64 n_blocks, const BatchTables& t, XBlock* __restrict__ xb,
                             u32* __restrict__ scratch, u8* __restrict__ out, int retry) {
    u64 bi_ = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (bi_ >= n_blocks) return;
    XBlock B = xb[bi_];
    if (retry) {
        if (!B.ovf) return;
        out += t.xdoc[B.doc].restage0;
    }
    const DocInfo& di = docs[B.doc];
    const u32 P = di.P, K = di.K, C = di.C;
    u32* sc = scratch + B.scratch;
    XReg peers, keys, cids;
    peers.ord = sc; peers.inv = sc + P;
    keys.ord = sc + 2 * P; keys.inv = keys.ord + K;
    cids.ord = keys.ord + 2 * K; cids.inv = cids.ord + C;
    u32* c_cidx = cids.ord + 2 * C;            // op columns, capacity n_rows each
    u32* c_prop = c_cidx + B.n_rows;
    u32* c_vt = c_prop + B.n_rows;
    u32* c_atoms = c_vt + B.n_rows;
    u32* d_peer = c_atoms + B.n_rows;          // delete columns, capacity n_dels each
    u32* d_ctr = d_peer + B.n_dels;
    u32* d_len = d_ctr + B.n_dels;
    const bool has_tree = (t.xdoc[B.doc].flags & 2u) != 0;
    const bool has_maps = (t.xdoc[B.doc].flags & 4u) != 0;
    u32* p_rank = d_len + B.n_dels;            // tree documents only (capacity n_rows): sorted distinct position ranks
    const u64 pos_lo = has_tree ? t.blocks[di.b0].pos0 : 0;
    // local index of a fractional index inside this block's position register
    auto pos_local = [&](u32 gpos) -> u32 {
        u32 r = t.pos_rank[gpos];
        u32 lo = 0, hi = B.n_pos;
        while (lo < hi) { u32 mid = (lo + hi) >> 1; if (p_rank[mid] < r) lo = mid + 1; else hi = mid; }
        return lo;
    };
    // doc-level peer index + counter of a tree op's subject / parent
    // bytes of one RawTreeMove value (value.rs write_raw_tree_move): subject, position, parent
    auto w_tree_value = [&](XSink& s, u32 ti) {
        uint4 ids = t.tr_ids[ti];
        u32 pk = ids.z & 3u;
        s.varint(peers.inv[ids.x]);
        s.varint(ids.y);
        s.varint(pk == TRP_DELETED ? 0u : pos_local(t.tr_pos[ti]));
        s.put(pk == TRP_ROOT ? 1 : 0);
        if (pk != TRP_ROOT) { s.varint(peers.inv[ids.z >> 2]); s.varint(ids.w); }
    };
    const u32 fc0 = B.fc0, N = B.fc1 - B.fc0;
    const u32 first_src = t.fc_src[fc0];
    u32 n_dep = 0;
    for (u32 j = 0; j < N; j++) n_dep += t.fc_from[fc0 + j] ? 0u : t.ch_ndeps[t.fc_src[fc0 + j]];
    for (u32 i = 0; i < P; i++) peers.inv[i] = 0xFFFFFFFFu;
    for (u32 i = 0; i < K; i++) keys.inv[i] = 0xFFFFFFFFu;
    for (u32 i = 0; i < C; i++) cids.inv[i] = 0xFFFFFFFFu;
    peers.n = keys.n = cids.n = 0;
    peers.reg(t.peer_map[t.blocks[t.ch_block[first_src]].peer0]);   // the author of the block's changes
    B.n_pos = 0;
    if (has_tree) {
        // position register, pre-filled in sorted order (block_encode.rs:156-178): ranks of the block's create /
        // move ops, heap-sorted, duplicates dropped
        u32 m = 0;
        for (u32 j = 0; j < N; j++) {
            XRows it(t, t.fc_pos[fc0 + j], t.fc_r0[fc0 + j]);
            u32 left = t.fc_nrows[fc0 + j];
            while (left) {
                uint4 r = xr_rec(t, it.row());
                if ((r.x & 7u) == XK_TREE && t.tr_pos[r.w] != 0xFFFFFFFFu) p_rank[m++] = t.pos_rank[t.tr_pos[r.w]];
                left--;
                if (left) it.next();
            }
        }
        auto sift = [&](u32 root, u32 end) {
            while (true) {
                u32 c = 2 * root + 1;
                if (c >= end) break;
                if (c + 1 < end && p_rank[c + 1] > p_rank[c]) c++;
                if (p_rank[root] >= p_rank[c]) break;
                u32 tmp = p_rank[root]; p_rank[root] = p_rank[c]; p_rank[c] = tmp;
                root = c;
            }
        };
        for (u32 i = m / 2; i-- > 0;) sift(i, m);
        for (u32 e = m; e-- > 1;) { u32 tmp = p_rank[0]; p_rank[0] = p_rank[e]; p_rank[e] = tmp; sift(0, e); }
        u32 w = 0;
        for (u32 i = 0; i < m; i++) if (i == 0 || p_rank[i] != p_rank[w - 1]) p_rank[w++] = p_rank[i];
        B.n_pos = w;
    }
    // ops in order: containers, map keys, delete targets (block_encode.rs:180-236).  The values section is written
    // on the way, at the start of the staging slot: the op's value prefix once its rows are merged, then the
    // payloads of those rows, which were just loaded
    XSink vs(out + B.stage, B.stage_cap);
    u32 n_ops = 0, n_del = 0;
    u32 prev_cidx = 0, prev_prop = 0, prev_dp = 0, prev_dc = 0, prev_dl = 0;   // 32-bit wrap-around deltas
    for (u32 j = 0; j < N; j++) {
        XRows it(t, t.fc_pos[fc0 + j], t.fc_r0[fc0 + j]);
        u32 left = t.fc_nrows[fc0 + j];
        u32 skip = t.fc_skip[fc0 + j];   // the first op of a change cut in front
        while (left) {
            XRows it0 = it;
            const u32 left0 = left;
            const u32 skip0 = skip;
            XOp o = xop_gather(t, di, it, left, skip);
            // the last op of a change cut at the end (fc_tail is loaded here only: a value held across the loop would
            // cost the encoder registers)
            if (CUT && !left) xop_slice_back(t, o, it.row(), t.fc_tail[fc0 + j]);
            skip = left ? it.skip : 0u;   // (the next op may start on the first kept row of a trimmed change)
            if (o.xk == XK_LIST) { vs.put(7); vs.varint(o.atoms); }
            else if (o.xk == XK_TEXT) vs.varint(o.f1 - o.f0);
            // DeltaRle columns are stored as deltas right away (the encoders then read every value once)
            u32 lc = cids.reg(o.cidx);
            u32 lp = (o.xk == XK_MAPSET || o.xk == XK_MAPDEL) ? keys.reg((u32)o.prop) : (u32)o.prop;
            if (o.xk == XK_LIST || o.xk == XK_TEXT || o.xk == XK_MAPSET) {
                // payloads after the op's own registrations: nested keys register in value order
                u32 k = left0 - left;
                while (k) {
                    const u8* pp;
                    u32 pn;
                    const u32 sk = k == left0 - left ? skip0 : it0.skip;
                    xr_payload_skip(t, it0.row(), o.xk, sk, &pp, &pn);
                    if (CUT && k == 1 && !left && t.fc_tail[fc0 + j]) xr_payload_drop_tail(o.xk, xr_len(t, it0.row()) - sk, t.fc_tail[fc0 + j], pp, &pn);
                    if (has_maps && o.xk != XK_TEXT) xvalue_copy(vs, pp, pn, t, t.blocks[t.ch_block[it0.ch]].key0, keys);
                    else vs.copy(pp, pn);
                    k--;
                    if (k) it0.next();
                }
            }
            c_cidx[n_ops] = lc - prev_cidx; prev_cidx = lc;
            c_prop[n_ops] = lp - prev_prop; prev_prop = lp;
            c_vt[n_ops] = xk_value_type(o.xk);
            c_atoms[n_ops] = o.atoms;
            if (o.xk == XK_TREE) {      // encode_tree_op (block_encode.rs:324-362): subject peer, then parent peer
                uint4 ids = t.tr_ids[o.f0];
                peers.reg(ids.x);
                if ((ids.z & 3u) != TRP_ROOT) peers.reg(ids.z >> 2);
                w_tree_value(vs, o.f0);
            }
            if (o.xk == XK_DEL) {
                u32 dp = peers.reg(o.f0);
                d_peer[n_del] = dp - prev_dp; prev_dp = dp;
                d_ctr[n_del] = o.f1 - prev_dc; prev_dc = o.f1;
                d_len[n_del] = (u32)o.f2 - prev_dl; prev_dl = (u32)o.f2;
                n_del++;
            }
            n_ops++;
        }
    }
    B.n_ops = n_ops;
    B.n_del_ops = n_del;
    B.sec_len[7] = (u32)vs.n;   // values section: written with the gather
    // ContainerArena::from_containers (arena.rs:103-147): roots register their name, normals their peer
    for (u32 i = 0; i < cids.n; i++) {
        const DocContainer& dc = t.dcont[di.cid0 + cids.ord[i]];
        if (dc.is_root) keys.reg(dc.key_or_peer); else peers.reg(dc.key_or_peer);
    }
    // encode_changes (block_meta_encode.rs:13-88): dependency peers
    for (u32 j = 0; j < N; j++) {
        if (t.fc_from[fc0 + j]) continue;
        u32 src = t.fc_src[fc0 + j];
        const BlockInfo& sb = t.blocks[t.ch_block[src]];
        for (u32 k = 0; k < t.ch_ndeps[src]; k++) peers.reg(t.peer_map[sb.peer0 + t.dep_peer_idx[t.ch_dep0[src] + k]]);
    }

    // ------------------------------------------------------------------ section writers (count or write)
    auto dep_self = [&](u32 j) -> bool { return t.fc_from[fc0 + j] ? true : t.ch_dep_self[t.fc_src[fc0 + j]] != 0; };
    auto dep_local = [&](XDeps& dc, u32 i) -> i64 {
        u64 di_ = dc.at(i);
        const BlockInfo& sb = t.blocks[t.ch_block[t.fc_src[fc0 + dc.j]]];
        return (i64)peers.inv[t.peer_map[sb.peer0 + t.dep_peer_idx[di_]]];
    };
    auto lamport = [&](u32 j) -> i64 { return (i64)t.ch_lamport[t.fc_src[fc0 + j]] + t.fc_from[fc0 + j]; };
    auto w_header = [&](XSink& s) {
        s.varint(peers.n);
        for (u32 i = 0; i < peers.n; i++) {
            u64 id = t.dpeer[di.peer0 + peers.ord[i]].id;
            for (int k = 0; k < 8; k++) s.put((u8)(id >> (8 * k)));
        }
        for (u32 j = 0; j + 1 < N; j++) s.varint(t.fc_atoms[fc0 + j]);
        enc_boolrle(s, N, dep_self);
        { XDeps dc(t, fc0, N); enc_anyrle(s, N, [&](u32 j) -> i64 { return (i64)dc.nd(j); }, WrVarint()); }
        { XDeps dc(t, fc0, N); enc_anyrle(s, n_dep, [&](u32 i) -> i64 { return dep_local(dc, i); }, WrVarint()); }
        { XDeps dc(t, fc0, N); enc_dod(s, n_dep, [&](u32 i) -> i64 { return (i64)t.dep_counter[dc.at(i)]; }); }
        enc_dod(s, N - 1, lamport);
    };
    auto w_meta = [&](XSink& s) {
        enc_dod(s, N, [&](u32 j) -> i64 { return t.ch_ts[t.fc_src[fc0 + j]]; });
        enc_anyrle(s, N, [&](u32 j) -> i64 { return (i64)t.ch_msg_len[t.fc_src[fc0 + j]]; }, WrVarint());
        for (u32 j = 0; j < N; j++) {
            u32 src = t.fc_src[fc0 + j];
            s.copy(t.bytes + t.ch_msg_off[src], t.ch_msg_len[src]);
        }
    };
    auto w_cids = [&](XSink& s) {
        s.varint(cids.n);
        for (u32 i = 0; i < cids.n; i++) {
            const DocContainer& dc = t.dcont[di.cid0 + cids.ord[i]];
            s.varint(4);
            s.put(dc.is_root ? 1 : 0);
            s.put(dc.type);
            if (dc.is_root) { s.varint(0); s.zigzag((i64)keys.inv[dc.key_or_peer]); }
            else { s.varint(peers.inv[dc.key_or_peer]); s.zigzag((i64)dc.counter); }
        }
    };
    auto w_keys = [&](XSink& s) {
        for (u32 i = 0; i < keys.n; i++) {
            u32 k = keys.ord[i];
            s.varint(t.dkey_len[di.key0 + k]);
            s.copy(t.bytes + t.dkey_off[di.key0 + k], t.dkey_len[di.key0 + k]);
        }
    };
    // stored deltas are 32-bit differences of i32 / small u32 values: sign-extend to the true delta
    auto w_opcol = [&](XSink& s, int col) {
        switch (col) {
            case 0: enc_anyrle(s, n_ops, [&](u32 i) -> i64 { return (i64)(i32)c_cidx[i]; }, WrZigzag()); break;
            case 1: enc_anyrle(s, n_ops, [&](u32 i) -> i64 { return (i64)(i32)c_prop[i]; }, WrZigzag()); break;
            case 2: enc_anyrle(s, n_ops, [&](u32 i) -> i64 { return (i64)c_vt[i]; }, WrByte()); break;
            default: enc_anyrle(s, n_ops, [&](u32 i) -> i64 { return (i64)c_atoms[i]; }, WrVarint());
        }
    };
    auto w_delcol = [&](XSink& s, int col) {
        switch (col) {
            case 0: enc_anyrle(s, n_del, [&](u32 i) -> i64 { return (i64)(i32)d_peer[i]; }, WrZigzag()); break;
            case 1: enc_anyrle(s, n_del, [&](u32 i) -> i64 { return (i64)(i32)d_ctr[i]; }, WrZigzag()); break;
            default: enc_anyrle(s, n_del, [&](u32 i) -> i64 { return (i64)(i32)d_len[i]; }, WrZigzag());
        }
    };
    // PositionArena::from_positions + encode_v2 (arena.rs:168-183, 218-224): common prefix with the predecessor
    auto pos_bytes_of = [&](u32 i, const u8** pb) -> u32 { u32 g = t.pos_rep[pos_lo + p_rank[i]]; *pb = t.pos_pool + t.pos_off[g]; return t.pos_len[g]; };
    auto pos_common = [&](u32 i) -> u32 {
        if (i == 0) return 0;
        const u8 *a, *b;
        u32 la = pos_bytes_of(i - 1, &a), lb = pos_bytes_of(i, &b);
        u32 n = la < lb ? la : lb, k = 0;
        while (k < n && a[k] == b[k]) k++;
        return k;
    };
    auto w_poscol = [&](XSink& s, int col) {
        if (col == 0) enc_anyrle(s, B.n_pos, [&](u32 i) -> i64 { return (i64)pos_common(i); }, WrVarint());
        else {
            s.varint(B.n_pos);
            for (u32 i = 0; i < B.n_pos; i++) {
                const u8* pb;
                u32 pl = pos_bytes_of(i, &pb), c = pos_common(i);
                s.varint(pl - c);
                s.copy(pb + c, pl - c);
            }
        }
    };
    u32 counter_len = 0;
    for (u32 j = 0; j < N; j++) counter_len += t.fc_atoms[fc0 + j];
    u32 counter0 = (u32)t.ch_counter[first_src] + t.fc_from[fc0];
    u32 lam0 = (u32)lamport(0);
    u32 lam_len = (u32)lamport(N - 1) + t.fc_atoms[B.fc1 - 1] - lam0;
    // staged pieces: the values (written by the gather), then in blob order the five header varints, the bodies of
    // sections 0-3, the position columns, the op columns, the delete columns (k_exp_finish adds the prefixes)
    XSink s(out + B.stage, B.stage_cap);
    s.n = B.sec_len[7];
    s.varint(counter0);
    s.varint(counter_len);
    s.varint(lam0);
    s.varint(lam_len);
    s.varint(N);
    u64 m = s.n;
    w_header(s); B.sec_len[0] = (u32)(s.n - m); m = s.n;
    w_meta(s); B.sec_len[1] = (u32)(s.n - m); m = s.n;
    w_cids(s); B.sec_len[2] = (u32)(s.n - m); m = s.n;
    w_keys(s); B.sec_len[3] = (u32)(s.n - m); m = s.n;
    u32 tot = 0;
    if (B.n_pos) {
        tot = 2;   // varint(1) varint(2)
        for (int c = 0; c < 2; c++) { w_poscol(s, c); B.col_len[7 + c] = (u32)(s.n - m); m = s.n; tot += varint_len(B.col_len[7 + c]) + B.col_len[7 + c]; }
    }
    B.sec_len[4] = tot;
    tot = 2;   // varint(1) varint(4)
    for (int c = 0; c < 4; c++) { w_opcol(s, c); B.col_len[c] = (u32)(s.n - m); m = s.n; tot += varint_len(B.col_len[c]) + B.col_len[c]; }
    B.sec_len[5] = tot;
    if (n_del) {
        tot = 2;
        for (int c = 0; c < 3; c++) { w_delcol(s, c); B.col_len[4 + c] = (u32)(s.n - m); m = s.n; tot += varint_len(B.col_len[4 + c]) + B.col_len[4 + c]; }
        B.sec_len[6] = tot;
    } else B.sec_len[6] = 0;
    B.ovf |= s.n > s.cap;   // still set after the retry: k_exp_finish then reads the retry slot
    u32 len = varint_len(counter0) + varint_len(counter_len) + varint_len(lam0) + varint_len(lam_len) + varint_len(N);
    for (int i = 0; i < 8; i++) len += varint_len(B.sec_len[i]) + B.sec_len[i];
    B.len = len;
    xb[bi_] = B;
}

template <int CAPPED> __global__ void k_exp_encode(const DocInfo* __restrict__ docs, u64 n_blocks, const __grid_constant__ BatchTables t, XBlock* __restrict__ xb,
                                                 u32* __restrict__ scratch, u8* __restrict__ out, int retry);
template <> __global__ void k_exp_encode<0>(const DocInfo* __restrict__ docs, u64 n_blocks, const __grid_constant__ BatchTables t, XBlock* __restrict__ xb,
                                            u32* __restrict__ scratch, u8* __restrict__ out, int retry) {
    exp_encode_body<0>(docs, n_blocks, t, xb, scratch, out, retry);
}
template <> __global__ void __launch_bounds__(64, 5) k_exp_encode<1>(const DocInfo* __restrict__ docs, u64 n_blocks, const __grid_constant__ BatchTables t,
                                                                     XBlock* __restrict__ xb, u32* __restrict__ scratch,
                                                                     u8* __restrict__ out, int retry) {
    exp_encode_body<0>(docs, n_blocks, t, xb, scratch, out, retry);
}
template <int CAPPED> __global__ void k_exp_encode_cut(const DocInfo* __restrict__ docs, u64 n_blocks, const __grid_constant__ BatchTables t, XBlock* __restrict__ xb,
                                                     u32* __restrict__ scratch, u8* __restrict__ out, int retry);
template <> __global__ void k_exp_encode_cut<0>(const DocInfo* __restrict__ docs, u64 n_blocks, const __grid_constant__ BatchTables t, XBlock* __restrict__ xb,
                                                u32* __restrict__ scratch, u8* __restrict__ out, int retry) {
    exp_encode_body<1>(docs, n_blocks, t, xb, scratch, out, retry);
}
template <> __global__ void __launch_bounds__(64, 5) k_exp_encode_cut<1>(const DocInfo* __restrict__ docs, u64 n_blocks, const __grid_constant__ BatchTables t,
                                                                         XBlock* __restrict__ xb, u32* __restrict__ scratch,
                                                                         u8* __restrict__ out, int retry) {
    exp_encode_body<1>(docs, n_blocks, t, xb, scratch, out, retry);
}

// thread per document, after the encode: block offsets inside the blob, blob length, and the blocks that outgrew their
// slot, each given a retry slot of its block length (an upper bound on its pieces) at a document-relative offset.  A
// document outside the request mask gets no blob (exp_len 0), so the buffer holds the requested blobs only.
__global__ void k_exp_layout(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t, XBlock* __restrict__ xb,
                             u32* __restrict__ padded_len, u32* __restrict__ n_ovf, u32* __restrict__ n_restage) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    XDoc& x = t.xdoc[d];
    u32 len = 0, ovf = 0, restage = 0;
    if (docs[d].code == DOC_OK && !(x.flags & 1) && (!t.x_req || t.x_req[d])) {
        len = 22;
        for (u32 i = 0; i < x.n_mb; i++) {
            XBlock& b = xb[x.ob0 + i];
            len += varint_len(b.len);
            b.off = len;
            len += b.len;
            if (b.ovf) {
                ovf++;
                b.stage = restage;
                b.stage_cap = b.len;
                restage += b.len;
            }
        }
    }
    x.exp_len = len;
    padded_len[d] = (len + 15u) & ~15u;
    n_ovf[d] = ovf;
    n_restage[d] = restage;
}

// warp per document: the blob from the staged pieces of its blocks (in the retry buffer for the blocks that outgrew
// their first slot) and their length prefixes, then header, mode, checksum (encoding.rs:397-416)
__global__ void k_exp_finish(const DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t, const XBlock* __restrict__ xb,
                             const u8* __restrict__ stage, const u8* __restrict__ restage, u8* __restrict__ out) {
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // warp per document: the checksum walks the whole blob
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const XDoc& x = t.xdoc[d];
    if (x.exp_len == 0) return;
    u8* b = out + x.exp_off;
    for (u32 i = 0; i < x.n_mb; i++) {
        const XBlock& B = xb[x.ob0 + i];
        u8* dst = b + B.off - varint_len(B.len);
        const u8* src = (B.ovf ? restage + x.restage0 : stage) + B.stage;
        u64 o = 0, so = B.sec_len[7];   // the values come first in the slot and last in the block
        auto prefix = [&](u32 v) {
            if (lane == 0) { XSink s(dst + o, ~0ull); s.varint(v); }
            o += varint_len(v);
        };
        auto piece = [&](u32 n) {   // four independent byte loads per lane in flight, then the stores
            u8* dd = dst + o;
            const u8* ss = src + so;
            u32 k = (u32)lane;
            for (; k + 96 < n; k += 128) {
                u8 a = ss[k], c = ss[k + 32], e = ss[k + 64], g = ss[k + 96];
                dd[k] = a; dd[k + 32] = c; dd[k + 64] = e; dd[k + 96] = g;
            }
            for (; k < n; k += 32) dd[k] = ss[k];
            o += n;
            so += n;
        };
        u32 head = B.len;   // the five header varints
        for (int k = 0; k < 8; k++) head -= varint_len(B.sec_len[k]) + B.sec_len[k];
        prefix(B.len);
        piece(head);
        for (int k = 0; k < 4; k++) { prefix(B.sec_len[k]); piece(B.sec_len[k]); }
        prefix(B.sec_len[4]);
        if (B.n_pos) {
            prefix(1); prefix(2);
            for (int c = 0; c < 2; c++) { prefix(B.col_len[7 + c]); piece(B.col_len[7 + c]); }
        }
        prefix(B.sec_len[5]);
        prefix(1); prefix(4);
        for (int c = 0; c < 4; c++) { prefix(B.col_len[c]); piece(B.col_len[c]); }
        prefix(B.sec_len[6]);
        if (B.n_del_ops) {
            prefix(1); prefix(3);
            for (int c = 0; c < 3; c++) { prefix(B.col_len[4 + c]); piece(B.col_len[4 + c]); }
        }
        prefix(B.sec_len[7]);
        so = 0;
        piece(B.sec_len[7]);
    }
    __syncwarp();
    if (lane == 0) {
        b[0] = 'l'; b[1] = 'o'; b[2] = 'r'; b[3] = 'o';
        for (int i = 4; i < 20; i++) b[i] = 0;
        b[20] = 0; b[21] = 4;   // FastUpdates, big endian
    }
    __syncwarp();
    u32 h = xxh32_warp(b + 20, x.exp_len - 20, XX_SEED_LORO, lane);
    if (lane == 0) { b[16] = (u8)h; b[17] = (u8)(h >> 8); b[18] = (u8)(h >> 16); b[19] = (u8)(h >> 24); }
}
