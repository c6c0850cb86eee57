// loro_b200 -- phase 6: deep-value materialisation (LoroDoc::get_deep_value as serde_json text).
//
// Replaces (reference): crates/loro-internal/src/state.rs:894-924 get_deep_value, :1039
//   get_container_deep_value ; state/{list,map,richtext}_state.rs value extraction ;
//   crates/loro-common/src/value.rs:692-711 (human-readable serde: I64 integer, Binary array, ...).
// Object keys are emitted in ascending byte order (the reference's FxHashMap order is unspecified;
// its own tests compare parsed JSON).  Round-1 shape: one thread per document, two passes over the same
// emitter (count bytes, then write) with an explicit frame stack instead of recursion.
#pragma once
#include "lb_tables.cuh"
#include "k_frame.cuh"
#include "k_tree.cuh"
#include "lb_f64.cuh"

struct Sink {
    u8* dst;   // nullptr = counting pass
    u64 n;
    u32 flags; // bit0: value the emitter cannot print exactly (non-integral f64, nested map value)
    bool wr;   // this lane writes (one warp per document: lane 0 owns the sequential parts)
    __device__ __forceinline__ void put(u8 c) { if (dst && wr) dst[n] = c; n++; }
    __device__ __forceinline__ void puts_(const char* s) { while (*s) put((u8)*s++); }
    __device__ void put_u64(u64 v) {
        char tmp[24];
        int k = 0;
        do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
        while (k) put((u8)tmp[--k]);
    }
    __device__ void put_i64(i64 v) {
        if (v < 0) { put('-'); put_u64((u64)(-(v + 1)) + 1); }
        else put_u64((u64)v);
    }
    // serde_json string escaping
    __device__ void put_escaped(const u8* s, u64 len) {
        const char* hex = "0123456789abcdef";
        for (u64 i = 0; i < len; i++) {
            u8 c = s[i];
            switch (c) {
                case '"': put('\\'); put('"'); break;
                case '\\': put('\\'); put('\\'); break;
                case '\b': put('\\'); put('b'); break;
                case '\f': put('\\'); put('f'); break;
                case '\n': put('\\'); put('n'); break;
                case '\r': put('\\'); put('r'); break;
                case '\t': put('\\'); put('t'); break;
                default:
                    if (c < 0x20) { put('\\'); put('u'); put('0'); put('0'); put((u8)hex[c >> 4]); put((u8)hex[c & 15]); }
                    else put(c);
            }
        }
    }
};

enum { FK_LIST = 1, FK_MAP = 2, FK_VLIST = 3, FK_VMAP = 4, FK_ROOT = 5, FK_TREE = 6 };
struct Frame {
    u8 kind;
    u8 first;      // nothing emitted yet at this level
    u8 cdepth;     // container levels down to this frame's (FK_ROOT 0, a root container 1; a value frame: its owner's)
    u8 vdepth;     // value levels down to this frame (0 but for FK_V*)
    u32 a, b, c;   // FK_LIST: cidx, run, elem-in-run ; FK_MAP/FK_ROOT: cidx, last key/root (or NONE) ; FK_V*: remaining
                   // FK_TREE: cidx, slot whose children are being listed, next child index (id_peer: node whose meta
                   // map was just printed, or NONE)
    const u8* p;   // value cursor (FK_LIST: inside the current run's payload ; FK_V*: nested items)
    u32 id_peer;   // doc peer idx + counter of the op atom that owns the values being printed
    i32 id_ctr;
};
// every frame but the root's adds one container level or one value level, and each kind of level is bounded on its own
#define MAX_FRAMES (2 * LB_MAX_NESTING + 2)

// per warp: the document's first peers with their ids as decimal text (tree node ids are "<counter>@<peer>": two per node,
// and formatting a 64-bit peer id costs twenty 64-bit divisions -- done once per peer instead of twice per node)
#define TREE_TXT_PEERS 8
struct TreeEmitSmem {
    u32 base[TREE_TXT_PEERS], end[TREE_TXT_PEERS];
    u8 len[TREE_TXT_PEERS];
    u8 txt[TREE_TXT_PEERS][20];
};

struct Emitter {
    const BatchTables& t;
    const DocInfo& di;
    Sink& out;
    Frame st[MAX_FRAMES];
    int sp;
    u32 err;
    int lane;
    u32 cur_blk;   // block of the op whose value is being printed (nested map keys are block-local indices)
    TreeEmitSmem* tsm;
    __device__ Emitter(const BatchTables& t_, const DocInfo& di_, Sink& o, int lane_, TreeEmitSmem* tsm_) : t(t_), di(di_), out(o), sp(0), err(0), lane(lane_), cur_blk(0), tsm(tsm_) {}

    __device__ int cmp_bytes(const u8* a, u32 al, const u8* b, u32 bl) {
        u32 n = al < bl ? al : bl;
        for (u32 i = 0; i < n; i++)
            if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
        return al < bl ? -1 : (al > bl ? 1 : 0);
    }
    __device__ u32 find_child(u64 peer_id, i32 ctr, u8 type) {
        for (u32 c = 0; c < di.C; c++) {
            const DocContainer& dc = t.dcont[di.cid0 + c];
            if (!dc.is_root && dc.type == type && dc.peer == peer_id && dc.counter == ctr) return c;
        }
        return 0xFFFFFFFFu;
    }
    __device__ void push(Frame f) {
        if (sp >= MAX_FRAMES) { err = LB_ERR(DOC_ERR_CAPACITY); return; }
        st[sp++] = f;
    }
    // bytes [*b0,*b1) of the payload of visible run r of a Text container (runs address unicode scalar values)
    __device__ const u8* text_run(const DocContainer& dc, u32 r, u64* b0, u64* b1) {
        u32 row = t.out_row[dc.out0 + r];
        u32 off = t.out_off[dc.out0 + r], len = t.out_len[dc.out0 + r];
        Cur c(t.bytes + t.op_val_off[row], t.op_val_len[row]);
        u64 blen = c.varint();
        const u8* s = c.p;
        *b0 = off;
        *b1 = off + len;
        if (blen != t.op_len[row]) {  // non-ASCII: map unicode offsets to byte offsets
            u64 i = 0, ch = 0;
            *b0 = blen;
            *b1 = blen;
            bool got0 = false;
            while (i <= blen) {
                if (ch == off && !got0) { *b0 = i; got0 = true; }
                if (ch == off + len) { *b1 = i; break; }
                if (i == blen) break;
                i++;
                while (i < blen && (s[i] & 0xC0) == 0x80) i++;
                ch++;
            }
        }
        return s;
    }
    // text of a Text container: concatenation of the visible runs; with many runs the lanes split them
    __device__ __noinline__ void emit_text(u32 cidx) {
        const DocContainer& dc = t.dcont[di.cid0 + cidx];
        out.put('"');
        if (dc.n_out >= 64) {
            u32 chunk = (dc.n_out + 31) / 32;
            u32 lo = (u32)lane * chunk, hi = lo + chunk < dc.n_out ? lo + chunk : dc.n_out;
            if (lo > dc.n_out) lo = dc.n_out;
            Sink cnt;
            cnt.dst = nullptr; cnt.n = 0; cnt.flags = 0; cnt.wr = false;
            for (u32 r = lo; r < hi; r++) {
                u64 b0, b1;
                const u8* s = text_run(dc, r, &b0, &b1);
                cnt.put_escaped(s + b0, b1 - b0);
            }
            u32 mine = (u32)cnt.n;
            u32 incl = (u32)warp_incl_scan((int)mine, lane);
            u32 total = __shfl_sync(LB_FULL, incl, 31);
            if (out.dst) {
                Sink w;
                w.dst = out.dst; w.n = out.n + (incl - mine); w.flags = 0; w.wr = true;
                for (u32 r = lo; r < hi; r++) {
                    u64 b0, b1;
                    const u8* s = text_run(dc, r, &b0, &b1);
                    w.put_escaped(s + b0, b1 - b0);
                }
            }
            __syncwarp();
            out.n += total;
        } else {
            for (u32 r = 0; r < dc.n_out; r++) {
                u64 b0, b1;
                const u8* s = text_run(dc, r, &b0, &b1);
                out.put_escaped(s + b0, b1 - b0);
            }
        }
        out.put('"');
    }
    // open a container value: scalars-like (text) print directly, list/map push a frame
    __device__ void open_container(u32 cidx, u8 type) {
        const u8 depth = st[sp - 1].cdepth + 1;
        if (depth > LB_MAX_NESTING + 1) { err = LB_ERR(DOC_ERR_UNSUPPORTED); return; }
        if (cidx == 0xFFFFFFFFu) {  // never targeted by an op: empty value of its type
            switch (type) {
                case CT_TEXT: out.puts_("\"\""); break;
                case CT_MAP: out.puts_("{}"); break;
                case CT_COUNTER: out.puts_("0.0"); break;
                default: out.puts_("[]");
            }
            return;
        }
        Frame f;
        f.first = 1;
        f.cdepth = depth;
        f.vdepth = st[sp - 1].vdepth;
        f.a = cidx;
        f.b = 0;
        f.c = 0;
        f.p = nullptr;
        f.id_peer = 0;
        f.id_ctr = 0;
        switch (type) {
            case CT_TEXT: emit_text(cidx); return;
            case CT_LIST: out.put('['); f.kind = FK_LIST; push(f); return;
            case CT_MAP: out.put('{'); f.kind = FK_MAP; f.b = 0xFFFFFFFFu; push(f); return;
            case CT_TREE:
                out.put('[');
                if (!di.has_tree) { out.put(']'); return; }   // no applied tree op in the document: no node tables
                if (di.has_tree & 2u) { emit_tree_parallel(cidx); out.put(']'); return; }
                f.kind = FK_TREE; f.b = (u32)di.atom_total + cidx; f.c = 0; f.id_peer = 0xFFFFFFFFu; push(f);
                return;
            default: out.puts_("null"); return;
        }
    }
    // "<counter>@<peer>" of the node stored at atom `a` (ID display: loro-common/src/id.rs:22-26)
    __device__ __noinline__ void put_tree_id_to(Sink& o, u32 a) {
        u32 p = 0;
        for (u32 q = 0; q < di.P; q++) {
            const DocPeer& dp = t.dpeer[di.peer0 + q];
            if (a >= dp.atom_base && a < dp.atom_base + (u32)dp.end_counter) { p = q; break; }
        }
        const DocPeer& dp = t.dpeer[di.peer0 + p];
        o.put('"');
        o.put_u64(a - dp.atom_base);
        o.put('@');
        o.put_u64(dp.id);
        o.put('"');
    }
    __device__ void put_tree_id(u32 a) { put_tree_id_to(out, a); }
    __device__ void put_fractional_index(Sink& o, u32 pos) {
        const char* HEX = "0123456789ABCDEF";   // crates/fractional_index/src/lib.rs:195-205
        const u8* pb = t.pos_pool + t.pos_off[pos];
        u32 pl = t.pos_len[pos];
        for (u32 k = 0; k < pl; k++) { o.put((u8)HEX[pb[k] >> 4]); o.put((u8)HEX[pb[k] & 15]); }
    }
    // n bytes of a thread-local buffer to global memory: single bytes up to the first 8-byte boundary, then whole words
    __device__ __noinline__ static void copy_out(u8* dst, const u8* src, u32 n) {
        u32 i = 0;
        while (i < n && ((uintptr_t)(dst + i) & 7)) { dst[i] = src[i]; i++; }
        for (; i + 8 <= n; i += 8) {
            u64 v = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) v |= (u64)src[i + q] << (8 * q);
            *(u64*)(dst + i) = v;
        }
        for (; i < n; i++) dst[i] = src[i];
    }
    __device__ __forceinline__ static void put_u32_to(Sink& o, u32 v) {   // 32-bit divisions by a constant: multiply + shift
        char tmp[10];
        int k = 0;
        do { tmp[k++] = (char)('0' + v % 10u); v /= 10u; } while (v);
        while (k) o.put((u8)tmp[--k]);
    }
    // "<counter>@<peer>" from the per-warp peer table (the caller checked di.P <= TREE_TXT_PEERS)
    __device__ __forceinline__ void put_tree_id_fast(Sink& o, u32 a) {
        u32 p = 0;
        for (u32 q = 0; q < di.P; q++) if (a >= tsm->base[q] && a < tsm->end[q]) { p = q; break; }
        o.put('"');
        put_u32_to(o, a - tsm->base[p]);
        o.put('@');
        for (u32 k = 0; k < tsm->len[p]; k++) o.put(tsm->txt[p][k]);
        o.put('"');
    }
    // every node of the hierarchy written by its own lane at the offsets k_tree_layout laid out (all meta maps empty);
    // the caller has printed '[' and prints ']'
    __device__ __noinline__ void emit_tree_parallel(u32 cidx) {
        const u64 tb = di.tree0;
        const u32 A = (u32)di.atom_total, slot = A + cidx;
        const u64 tr_lo = t.blocks[di.b0].tr0;
        const u32 total = ((const u32*)(t.ns_key + tb))[slot];
        if (out.dst) {
            const bool fast = di.P <= TREE_TXT_PEERS;
            if (fast) {
                __syncwarp();
                if ((u32)lane < di.P) {
                    const DocPeer& dp = t.dpeer[di.peer0 + lane];
                    tsm->base[lane] = dp.atom_base;
                    tsm->end[lane] = dp.atom_base + (u32)dp.end_counter;
                    char tmp[20];
                    int k = 0;
                    u64 v = dp.id;
                    do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
                    tsm->len[lane] = (u8)k;
                    for (int i = 0; i < k; i++) tsm->txt[lane][i] = (u8)tmp[k - 1 - i];
                }
                __syncwarp();
            }
            const u64 start = out.n - 1;   // the container's '['
            for (u32 a = (u32)lane; a < A; a += 32) {
                if (t.tn_root[tb + a] != slot) continue;
                // the node's two pieces are composed in a thread-local buffer and leave as 8-byte stores: byte stores
                // of 32 lanes into 32 different sectors were the whole cost of this kernel (6.5 GB of JSON in config C5)
                u8 buf[216];
                const u32 pos = t.tr_rec[tr_lo + t.tn_move[tb + a]].z;
                const bool direct = t.pos_len[pos] > 32;     // an unusually long fractional index: write in place
                Sink w;
                w.flags = 0; w.wr = true;
                w.dst = direct ? out.dst + start + t.tn_aopen[tb + a] : buf;
                w.n = 0;
                u32 sib = t.tn_sib[tb + a], par = t.tn_parent[tb + a];
                if (sib) w.put(',');
                w.puts_("{\"children\":[");
                if (!direct) copy_out(out.dst + start + t.tn_aopen[tb + a], buf, (u32)w.n);
                w.dst = direct ? out.dst + start + t.tn_aclose[tb + a] : buf;
                w.n = 0;
                w.puts_("],\"fractional_index\":\"");
                put_fractional_index(w, pos);
                w.puts_("\",\"id\":");
                if (fast) put_tree_id_fast(w, a); else put_tree_id_to(w, a);
                w.puts_(",\"index\":");
                put_u32_to(w, sib);
                w.puts_(",\"meta\":{},\"parent\":");
                if (par == TREE_ROOT) w.puts_("null");
                else if (fast) put_tree_id_fast(w, par);
                else put_tree_id_to(w, par);
                w.put('}');
                if (!direct) copy_out(out.dst + start + t.tn_aclose[tb + a], buf, (u32)w.n);
            }
            __syncwarp();
        }
        out.n += total;
    }
    // one step of the hierarchy walk (state/tree_state.rs:814-831 get_all_hierarchy_nodes_under + :1424-1452
    // TreeNodeWithChildren::into_value, keys in ascending order): no per-level frames -- the walk climbs back
    // through the parent links
    __device__ __noinline__ void tree_step(Frame& f) {
        const u64 tb = di.tree0;
        const u32 A = (u32)di.atom_total;
        const u64 tr_lo = t.blocks[di.b0].tr0;
        if (f.id_peer != 0xFFFFFFFFu) {
            // the meta map of node f.id_peer has been printed: close the node, continue with its next sibling
            u32 node = f.id_peer;
            f.id_peer = 0xFFFFFFFFu;
            u32 par = t.tn_parent[tb + node];
            out.puts_(",\"parent\":");
            if (par == TREE_ROOT) out.puts_("null"); else put_tree_id(par);
            out.put('}');
            f.b = par == TREE_ROOT ? A + f.a : par;
            f.c = t.tn_sib[tb + node] + 1;
            return;
        }
        u32 slot = f.b;
        if (f.c < t.tn_cnt[tb + slot]) {   // open the next child
            u32 node = t.tn_child[tb + t.tn_base[tb + slot] + f.c];
            if (f.c) out.put(',');
            out.puts_("{\"children\":[");
            f.b = node;
            f.c = 0;
            return;
        }
        out.put(']');
        if (slot >= A) { sp--; return; }   // back at the container's root list: done
        // children of node `slot` are done: the rest of its object
        u32 node = slot;
        uint4 rec = t.tr_rec[tr_lo + t.tn_move[tb + node]];
        out.puts_(",\"fractional_index\":\"");
        put_fractional_index(out, rec.z);
        out.puts_("\",\"id\":");
        put_tree_id(node);
        out.puts_(",\"index\":");
        out.put_u64(t.tn_sib[tb + node]);
        out.puts_(",\"meta\":");
        // TreeID::associated_meta_container: the Map whose id is the node's id
        u32 p = 0;
        for (u32 q = 0; q < di.P; q++) {
            const DocPeer& dp = t.dpeer[di.peer0 + q];
            if (node >= dp.atom_base && node < dp.atom_base + (u32)dp.end_counter) { p = q; break; }
        }
        const DocPeer& dp = t.dpeer[di.peer0 + p];
        f.id_peer = node;
        int my = sp - 1;
        open_container(find_child(dp.id, (i32)(node - dp.atom_base), CT_MAP), CT_MAP);
        (void)my;
    }
    // print a scalar LoroValue (kinds 0-6) at *pp into `o`; false (nothing consumed) for lists, maps, containers
    __device__ bool emit_scalar(Sink& o, const u8** pp, const u8* end) {
        Cur c(*pp, (size_t)(end - *pp));
        u8 kind = c.get();
        switch (kind) {
            case 0: o.puts_("null"); break;
            case 1: o.puts_("true"); break;
            case 2: o.puts_("false"); break;
            case 3: o.put_i64(c.sleb()); break;
            case 4: {
                u64 bits = 0;
                for (int i = 0; i < 8; i++) bits = (bits << 8) | c.get();
                char buf[32];   // shortest round-trip text, as serde_json (ryu) prints it: lb_f64.cuh
                int n = f64_format(bits, buf);
                for (int i = 0; i < n; i++) o.put((u8)buf[i]);
                break;
            }
            case 5: {
                u64 n = c.varint();
                o.put('"');
                o.put_escaped(c.p, n <= c.left() ? n : c.left());
                o.put('"');
                c.skip(n);
                break;
            }
            case 6: {
                u64 n = c.varint();
                o.put('[');
                for (u64 i = 0; i < n && !c.err; i++) {
                    if (i) o.put(',');
                    o.put_u64(c.get());
                }
                o.put(']');
                break;
            }
            default: return false;
        }
        if (c.err) err = LB_ERR(DOC_ERR_CORRUPT);
        *pp = c.p;
        return true;
    }
    // print the LoroValue at *pp (kind byte + content), advancing *pp; may push a frame
    __device__ void emit_value(const u8** pp, const u8* end, u32 id_peer, i32 id_ctr) {
        if (emit_scalar(out, pp, end)) return;
        Cur c(*pp, (size_t)(end - *pp));
        u8 kind = c.get();
        switch (kind) {
            case 7: case 8: {
                u64 n = c.varint();
                out.put(kind == 7 ? '[' : '{');
                Frame f;
                f.kind = kind == 7 ? FK_VLIST : FK_VMAP;
                f.first = 1;
                f.cdepth = st[sp - 1].cdepth;
                f.vdepth = st[sp - 1].vdepth + 1;   // the decoder admits no value deeper than LB_MAX_NESTING
                if (f.vdepth > LB_MAX_NESTING) { err = LB_ERR(DOC_ERR_UNSUPPORTED); return; }
                f.a = (u32)n;
                f.b = cur_blk;
                f.c = 0xFFFFFFFFu;   // FK_VMAP: block-local index of the last key printed
                f.p = c.p;
                f.id_peer = id_peer;
                f.id_ctr = id_ctr;
                *pp = c.p;  // the frame owns the cursor from here; caller re-syncs when the frame pops
                push(f);
                return;
            }
            case 9: {
                u8 type = c.get();
                *pp = c.p;
                u32 child = find_child(t.dpeer[di.peer0 + id_peer].id, id_ctr, type);
                open_container(child, type);
                return;
            }
            default:
#ifdef LB_SIMT_EMU
                if (getenv("LB_EMU_TRACE")) fprintf(stderr, "emit_value: bad kind %u (sp=%d top kind=%d)\n", kind, sp, sp ? st[sp-1].kind : -1);
#endif
                err = LB_ERR(DOC_ERR_CORRUPT);
        }
        if (c.err) err = LB_ERR(DOC_ERR_CORRUPT);
        *pp = c.p;
    }
    // pointer to the payload of list-insert row `row` positioned at element `skip`
    __device__ const u8* list_elem_ptr(u32 row, u32 skip, const u8** end) {
        Cur c(t.bytes + t.op_val_off[row], t.op_val_len[row]);
        (void)c.get();     // LoroValue kind byte (7 = List)
        (void)c.varint();  // element count
        for (u32 i = 0; i < skip && !c.err; i++) {
            u8 k = c.get();
            skip_loro_value_content(c, k, nullptr);
        }
        *end = c.end;
        return c.p;
    }

    // ---- one warp per document: the runs of a scalar-only list are split over the lanes (sizes, scan, write)
    __device__ __noinline__ bool coop_list(u32 cidx) {
        const DocContainer& dc = t.dcont[di.cid0 + cidx];
        u32 n_out = dc.n_out;
        if (n_out < 64) return false;
        u32 chunk = (n_out + 31) / 32;
        u32 lo = (u32)lane * chunk, hi = lo + chunk < n_out ? lo + chunk : n_out;
        if (lo > n_out) lo = n_out;
        Sink cnt;
        cnt.dst = nullptr; cnt.n = 0; cnt.flags = 0; cnt.wr = false;
        bool complex_ = false;
        u32 elems = 0;
        u32 err0 = err;   // a lane-local decode error must not leave the lanes in different states
        for (u32 r = lo; r < hi && !complex_; r++) {
            u32 row = t.out_row[dc.out0 + r];
            u32 off = t.out_off[dc.out0 + r], len = t.out_len[dc.out0 + r];
            const u8* end;
            const u8* p = list_elem_ptr(row, off, &end);
            for (u32 e = 0; e < len; e++) {
                if (!emit_scalar(cnt, &p, end)) { complex_ = true; break; }
                elems++;
            }
        }
        if (__any_sync(LB_FULL, complex_ || err != err0)) { err = err0; return false; }
        u32 mine = (u32)cnt.n + elems - (lane == 0 ? 1u : 0u);   // a comma before every element but the first
        u32 incl = (u32)warp_incl_scan((int)mine, lane);
        u32 total = __shfl_sync(LB_FULL, incl, 31);
        u32 flags_all = cnt.flags;
        for (int d = 16; d > 0; d >>= 1) flags_all |= __shfl_xor_sync(LB_FULL, flags_all, d);
        out.flags |= flags_all;
        if (out.dst) {
            Sink w;
            w.dst = out.dst; w.n = out.n + (incl - mine); w.flags = 0; w.wr = true;
            bool first = lane == 0;
            for (u32 r = lo; r < hi; r++) {
                u32 row = t.out_row[dc.out0 + r];
                u32 off = t.out_off[dc.out0 + r], len = t.out_len[dc.out0 + r];
                const u8* end;
                const u8* p = list_elem_ptr(row, off, &end);
                for (u32 e = 0; e < len; e++) {
                    if (!first) w.put(',');
                    first = false;
                    emit_scalar(w, &p, end);
                }
            }
        }
        __syncwarp();
        out.n += total;
        return true;
    }

    // one step of a nested LoroValue::Map (kept out of line: the walk is rare and register hungry)
    __device__ __noinline__ void vmap_step(Frame& f) {
            // LoroValue::Map inside a value (encoding/value.rs:1027-1036): entries = (key index into the block's
            // key arena, value).  Printed in ascending key order like every object here; of two entries with
            // the same key the later one wins.  Each step re-scans the entries for the next key.
            const BlockInfo& vb = t.blocks[f.b];
            const u8* best_val = nullptr;
            u32 best = 0xFFFFFFFFu;
            {
                Cur c(f.p, (size_t)(1u << 30));
                for (u32 i = 0; i < f.a && !c.err; i++) {
                    u64 ki = c.varint();
                    const u8* val = c.p;
                    u8 k = c.get();
                    skip_loro_value_content(c, k, nullptr);
                    if (ki >= vb.n_keys) { err = LB_ERR(DOC_ERR_CORRUPT); break; }
                    const u8* kb = t.bytes + t.key_off[vb.key0 + ki];
                    u32 kl = t.key_len[vb.key0 + ki];
                    if (f.c != 0xFFFFFFFFu &&
                        cmp_bytes(kb, kl, t.bytes + t.key_off[vb.key0 + f.c], t.key_len[vb.key0 + f.c]) <= 0) continue;
                    if (best == 0xFFFFFFFFu ||
                        cmp_bytes(kb, kl, t.bytes + t.key_off[vb.key0 + best], t.key_len[vb.key0 + best]) <= 0) { best = (u32)ki; best_val = val; }
                }
                if (c.err) err = LB_ERR(DOC_ERR_CORRUPT);
            }
            if (err) return;
            if (best == 0xFFFFFFFFu) { out.put('}'); sp--; return; }
            if (!f.first) out.put(',');
            f.first = 0;
            f.c = best;
            out.put('"');
            out.put_escaped(t.bytes + t.key_off[vb.key0 + best], t.key_len[vb.key0 + best]);
            out.put('"');
            out.put(':');
            cur_blk = f.b;
            const u8* p = best_val;
            emit_value(&p, p + (1u << 30), f.id_peer, f.id_ctr);
    }
    __device__ void run(void) {
        // root frame: iterate root containers in ascending name order
        out.put('{');
        Frame rf;
        rf.kind = FK_ROOT;
        rf.first = 1;
        rf.cdepth = 0;
        rf.vdepth = 0;
        rf.a = 0;
        rf.b = 0xFFFFFFFFu;
        rf.c = 0;
        rf.p = nullptr;
        rf.id_peer = 0;
        rf.id_ctr = 0;
        push(rf);
        int guard_parent_sync = 0;
        (void)guard_parent_sync;
        while (sp > 0 && !err) {
            Frame& f = st[sp - 1];
            switch (f.kind) {
                case FK_ROOT: {
                    // next root name greater than the previous one (ties: highest container index wins)
                    u32 best = 0xFFFFFFFFu;
                    for (u32 c = 0; c < di.C; c++) {
                        const DocContainer& dc = t.dcont[di.cid0 + c];
                        if (!dc.is_root) continue;
                        if (f.b != 0xFFFFFFFFu) {
                            const DocContainer& pc = t.dcont[di.cid0 + f.b];
                            if (cmp_bytes(t.bytes + dc.name_off, dc.name_len, t.bytes + pc.name_off, pc.name_len) <= 0) continue;
                        }
                        if (best == 0xFFFFFFFFu) best = c;
                        else {
                            const DocContainer& bc = t.dcont[di.cid0 + best];
                            int cm = cmp_bytes(t.bytes + dc.name_off, dc.name_len, t.bytes + bc.name_off, bc.name_len);
                            if (cm < 0 || cm == 0) best = c;
                        }
                    }
                    if (best == 0xFFFFFFFFu) { out.put('}'); sp--; break; }
                    if (!f.first) out.put(',');
                    f.first = 0;
                    f.b = best;
                    const DocContainer& dc = t.dcont[di.cid0 + best];
                    out.put('"');
                    out.put_escaped(t.bytes + dc.name_off, dc.name_len);
                    out.put('"');
                    out.put(':');
                    open_container(best, dc.type);
                    break;
                }
                case FK_LIST: {
                    const DocContainer& dc = t.dcont[di.cid0 + f.a];
                    if (f.first && f.b == 0 && f.c == 0 && coop_list(f.a)) { out.put(']'); sp--; break; }
                    if (f.b >= dc.n_out) { out.put(']'); sp--; break; }
                    u32 row = t.out_row[dc.out0 + f.b];
                    u32 off = t.out_off[dc.out0 + f.b], len = t.out_len[dc.out0 + f.b];
                    const u8* end;
                    if (f.c == 0 || f.p == nullptr) f.p = list_elem_ptr(row, off + f.c, &end);
                    else { Cur tmp(t.bytes + t.op_val_off[row], t.op_val_len[row]); end = tmp.end; }
                    if (!f.first) out.put(',');
                    f.first = 0;
                    u32 id_peer = t.ch_peer[t.op_change[row]];
                    i32 id_ctr = t.op_counter[row] + (i32)(off + f.c);
                    // advance the frame *before* emitting: emit_value may push a child frame
                    const u8* p = f.p;
                    f.c++;
                    bool run_done = f.c >= len;
                    int my = sp - 1;
                    cur_blk = t.ch_block[t.op_change[row]];
                    emit_value(&p, end, id_peer, id_ctr);
                    // a pushed nested-value frame consumes bytes we cannot see here; re-derive the cursor lazily
                    if (sp - 1 != my) st[my].p = nullptr; else st[my].p = p;
                    if (run_done) { st[my].b++; st[my].c = 0; st[my].p = nullptr; }
                    break;
                }
                case FK_MAP: {
                    // next key (ascending bytes) with a live winner
                    u32 best = 0xFFFFFFFFu;
                    for (u32 k = 0; k < di.K; k++) {
                        u64 slot = di.mapslot0 + (u64)f.a * di.K + k;
                        if (t.map_best[slot] == 0) continue;
                        u32 row = t.map_row[slot];
                        if (t.op_kind[row] != OPK_MAP_SET) continue;
                        const u8* kb = t.bytes + t.dkey_off[di.key0 + k];
                        u32 kl = t.dkey_len[di.key0 + k];
                        if (f.b != 0xFFFFFFFFu &&
                            cmp_bytes(kb, kl, t.bytes + t.dkey_off[di.key0 + f.b], t.dkey_len[di.key0 + f.b]) <= 0) continue;
                        if (best == 0xFFFFFFFFu ||
                            cmp_bytes(kb, kl, t.bytes + t.dkey_off[di.key0 + best], t.dkey_len[di.key0 + best]) < 0) best = k;
                    }
                    if (best == 0xFFFFFFFFu) { out.put('}'); sp--; break; }
                    if (!f.first) out.put(',');
                    f.first = 0;
                    f.b = best;
                    out.put('"');
                    out.put_escaped(t.bytes + t.dkey_off[di.key0 + best], t.dkey_len[di.key0 + best]);
                    out.put('"');
                    out.put(':');
                    u32 row = t.map_row[di.mapslot0 + (u64)f.a * di.K + best];
                    const u8* p = t.bytes + t.op_val_off[row];
                    cur_blk = t.ch_block[t.op_change[row]];
                    emit_value(&p, p + t.op_val_len[row], t.ch_peer[t.op_change[row]], t.op_counter[row]);
                    break;
                }
                case FK_VMAP: vmap_step(f); break;
                case FK_VLIST: {
                    if (f.a == 0) { out.put(']'); sp--; break; }
                    if (!f.first) out.put(',');
                    f.first = 0;
                    f.a--;
                    const u8* p = f.p;
                    const u8* end = p + (1u << 30);
                    int my = sp - 1;
                    // where the next sibling starts (a child frame may be pushed by emit_value)
                    {
                        Cur sk(p, (size_t)(1u << 30));
                        u8 k = sk.get();
                        skip_loro_value_content(sk, k, nullptr);
                        st[my].p = sk.p;
                    }
                    cur_blk = f.b;
                    emit_value(&p, end, f.id_peer, f.id_ctr);
                    break;
                }
                case FK_TREE: tree_step(f); break;
                default: err = LB_ERR(DOC_ERR_CAPACITY);
            }
        }
    }
};

// pass = 0: count bytes into docs[d].json_len ; pass = 1: write at docs[d].json_off
__global__ void __launch_bounds__(128, 8) k_json(DocInfo* __restrict__ docs, u32 n_docs, const __grid_constant__ BatchTables t, u8* __restrict__ json, int pass) {
    __shared__ TreeEmitSmem tsm[4];   // 128 threads: one entry per warp
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // one warp per document
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    DocInfo& di = docs[d];
    if (di.code != DOC_OK) { if (!pass && lane == 0) di.json_len = 0; return; }
    Sink s;
    s.dst = pass ? json + di.json_off : nullptr;
    s.n = 0;
    s.flags = 0;
    s.wr = lane == 0;
    Emitter e(t, di, s, lane, &tsm[(threadIdx.x >> 5) & 3]);
    e.run();
    __syncwarp();
    if (!pass && lane == 0) {
        di.json_len = (u32)s.n;
        if (e.err) di.code = e.err;
        else if (s.flags & 1) di.has_unsupported |= 0x80000000u;
    }
}

// thread per doc: padded length for the scan (JSON slots are 4-byte aligned for the hash kernel)
__global__ void k_json_padlen(const DocInfo* __restrict__ docs, u32 n_docs, u32* __restrict__ padded) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    padded[d] = (docs[d].json_len + 3u) & ~3u;
}

// warp per doc: order-independent state hash + counters
__global__ void k_doc_hash(const DocInfo* __restrict__ docs, u32 n_docs, const u8* __restrict__ json,
                           unsigned long long* __restrict__ acc /* [0]=hash xor, [1]=atom ops, [2]=pending, [3]=ok docs */) {
    u32 d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    if (di.code != DOC_OK) return;
    unsigned long long h = 0;
    if (json) h = ((unsigned long long)xxh32_warp(json + di.json_off, di.json_len, 0, lane) << 32) | di.json_len;
    if (lane) return;
    atomicXor(&acc[0], h);
    atomicAdd(&acc[1], (unsigned long long)di.atom_ops);
    atomicAdd(&acc[2], (unsigned long long)di.n_pending);
    atomicAdd(&acc[3], 1ull);
}
