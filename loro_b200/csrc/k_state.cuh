// loro_b200 -- phase 6: deep-value materialisation (LoroDoc::get_deep_value as serde_json text).
//
// Replaces (reference): crates/loro-internal/src/state.rs:894-924 get_deep_value, :1039
//   get_container_deep_value ; state/{list,map,richtext}_state.rs value extraction ;
//   crates/loro-common/src/value.rs:692-711 (human-readable serde: I64 integer, Binary array, ...).
// Object keys are emitted in ascending byte order (the reference's FxHashMap order is unspecified;
// its own tests compare parsed JSON).  One warp per document, two launches of the same emitter (count bytes, then
// write) with an explicit frame stack instead of recursion: lane 0 walks the document; the lanes share the elements of
// a scalar-only List or the runs of a Text with 64 runs or more (32 consecutive pieces at a time, staged in shared
// memory and stored as words) and the nodes of a Tree whose meta maps are empty.
#pragma once
#include "lb_tables.cuh"
#include "k_frame.cuh"
#include "k_tree.cuh"
#include "lb_f64.cuh"

// the text printers of a sink S, which supplies put(u8)
template <class S> struct PutText {
    __device__ __forceinline__ void put(u8 c) { static_cast<S*>(this)->put(c); }
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

struct Sink : PutText<Sink> {
    u8* dst;   // nullptr = counting pass
    u64 n;
    u32 flags; // bit0: value the emitter cannot print exactly (non-integral f64, nested map value)
    bool wr;   // this lane writes (one warp per document: lane 0 owns the sequential parts)
    __device__ __forceinline__ void put(u8 c) { if (dst && wr) dst[n] = c; n++; }
};

// Containers with many runs are written 32 pieces at a time (a list element or a text run per lane): each lane prints
// its piece into its slot, the warp packs the slots in lane order and stores the packed window with aligned words.
// 32 bytes hold every integer, float, bool and null with its comma, and a short string with its escapes; a longer
// piece is counted past its slot and written straight from its lane.
#define JSON_SLOT 32
struct JsonStage {
    u8 slot[32][JSON_SLOT + 1];   // odd stride: the lanes' byte stores at the same slot position hit different banks
    u32 packed[(32 * JSON_SLOT + 4) / 4];   // the window behind up to 3 bytes that put it on the global word grid
};
struct SlotSink : PutText<SlotSink> {
    u8* dst;
    u32 n;
    __device__ __forceinline__ void put(u8 c) { if (n < JSON_SLOT) dst[n] = c; n++; }
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
    JsonStage* stg;
    __device__ Emitter(const BatchTables& t_, const DocInfo& di_, Sink& o, int lane_, TreeEmitSmem* tsm_, JsonStage* stg_)
        : t(t_), di(di_), out(o), sp(0), err(0), lane(lane_), cur_blk(0), tsm(tsm_), stg(stg_) {}

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
    // text of a Text container: concatenation of the visible runs; with many runs, consecutive runs on consecutive lanes
    __device__ __noinline__ void emit_text(u32 cidx) {
        const DocContainer& dc = t.dcont[di.cid0 + cidx];
        out.put('"');
        if (dc.n_out >= 64) {
            Sink cnt;
            cnt.dst = nullptr; cnt.n = 0; cnt.flags = 0; cnt.wr = false;
            u64 pos = out.n;
            for (u32 r0 = 0; r0 < dc.n_out; r0 += 32) {
                const u32 r = r0 + (u32)lane;
                u64 b0 = 0, b1 = 0;
                const u8* s = r < dc.n_out ? text_run(dc, r, &b0, &b1) : nullptr;
                if (out.dst) {
                    SlotSink w;
                    w.dst = stg->slot[lane]; w.n = 0;
                    w.put_escaped(s + b0, b1 - b0);
                    const u32 incl = (u32)warp_incl_scan((int)w.n, lane), W = __shfl_sync(LB_FULL, incl, 31);
                    if (store_window(out.dst + pos, w.n, incl - w.n, W)) {
                        Sink d;
                        d.dst = out.dst + pos + (incl - w.n); d.n = 0; d.flags = 0; d.wr = true;
                        d.put_escaped(s + b0, b1 - b0);
                    }
                    pos += W;
                } else cnt.put_escaped(s + b0, b1 - b0);
            }
            __syncwarp();
            if (out.dst) out.n = pos;
            else out.n += (u32)warp_sum((int)cnt.n);
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
    template <class S> __device__ bool emit_scalar(S& o, const u8** pp, const u8* end) {
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

    // write pass of a container written 32 pieces at a time: this lane's piece of n bytes, printed into its slot as far
    // as it fits, goes to dst + off; the window is the W bytes at dst.  True when the piece outgrew its slot: the lane
    // then writes it itself.
    __device__ __noinline__ bool store_window(u8* dst, u32 n, u32 off, u32 W) {
        const bool big = n > JSON_SLOT;
        const u8* s = stg->slot[lane];
        if (__any_sync(LB_FULL, big)) {   // rare: every lane stores its own piece
            if (!big) for (u32 i = 0; i < n; i++) dst[off + i] = s[i];
            __syncwarp();
            return big;
        }
        const u32 mis = (u32)((uintptr_t)dst & 3), e = mis + W;
        u8* pk = (u8*)stg->packed;
        for (u32 i = 0; i < n; i++) pk[mis + off + i] = s[i];
        __syncwarp();
        u8* d0 = dst - mis;   // word aligned: packed word w goes to word w of d0
        for (u32 w = (u32)lane; 4 * w < e; w += 32) {
            const u32 lo = 4 * w;
            if (lo >= mis && lo + 4 <= e) ((u32*)d0)[w] = stg->packed[w];
            else for (u32 b = lo < mis ? mis : lo; b < lo + 4 && b < e; b++) d0[b] = pk[b];
        }
        __syncwarp();
        return false;
    }

    // ---- one warp per document: the elements of a scalar-only list, element k of each window of 32 on lane k % 32.
    // The runs are taken 32 at a time (consecutive runs on consecutive lanes), a warp scan of their lengths gives each
    // element its run; the count pass sums the printed lengths, the write pass prints every element once into its slot.
    __device__ __noinline__ bool coop_list(u32 cidx) {
        const DocContainer& dc = t.dcont[di.cid0 + cidx];
        const u32 n_out = dc.n_out;
        if (n_out < 64) return false;
        const u32 err0 = err;   // a lane-local decode error must not leave the lanes in different states
        Sink cnt;
        cnt.dst = nullptr; cnt.n = 0; cnt.flags = 0; cnt.wr = false;
        u64 pos = out.n;
        for (u32 r0 = 0; r0 < n_out; r0 += 32) {
            const u32 r = r0 + (u32)lane;
            u32 row = 0, off = 0, len = 0;
            if (r < n_out) { row = t.out_row[dc.out0 + r]; off = t.out_off[dc.out0 + r]; len = t.out_len[dc.out0 + r]; }
            const u32 incl = (u32)warp_incl_scan((int)len, lane), T = __shfl_sync(LB_FULL, incl, 31);
            const u8* carry = nullptr;   // where the element after the previous window starts
            for (u32 k0 = 0; k0 < T; k0 += 32) {
                const u32 k = k0 + (u32)lane;
                u32 j = 0;   // runs of the batch that end at or before element k
#pragma unroll
                for (u32 s = 16; s; s >>= 1) if (__shfl_sync(LB_FULL, incl, j + s - 1) <= k) j += s;
                const u32 jrow = __shfl_sync(LB_FULL, row, j), joff = __shfl_sync(LB_FULL, off, j);
                const u32 jstart = __shfl_sync(LB_FULL, incl - len, j);
                const u8* p = nullptr;
                const u8* el = nullptr;
                const u8* end = nullptr;
                const bool comma = r0 + k != 0;   // a comma before every element but the first
                bool ok = true;
                SlotSink w;
                w.dst = stg->slot[lane]; w.n = 0;
                if (k < T) {
                    end = t.bytes + t.op_val_off[jrow] + t.op_val_len[jrow];
                    u32 from = k0;   // a run that goes on from the previous window goes on from that window's cursor
                    if (jstart < k0) p = carry;
                    else { p = list_elem_ptr(jrow, joff, &end); from = jstart; }
                    Cur c(p, (size_t)(end - p));
                    for (u32 i = from; i < k && !c.err; i++) {
                        u8 kind = c.get();
                        skip_loro_value_content(c, kind, nullptr);
                    }
                    el = p = c.p;
                    if (out.dst) {
                        if (comma) w.put(',');
                        ok = emit_scalar(w, &p, end);
                    } else {
                        if (comma) cnt.put(',');
                        ok = emit_scalar(cnt, &p, end);
                    }
                }
                // a nested value: the sequential walk prints the container (over what earlier windows wrote, the same bytes)
                if (__any_sync(LB_FULL, !ok || err != err0)) { err = err0; return false; }
                carry = (const u8*)__shfl_sync(LB_FULL, (unsigned long long)p, 31);
                if (out.dst) {
                    const u32 n = k < T ? w.n : 0u;
                    const u32 wincl = (u32)warp_incl_scan((int)n, lane), W = __shfl_sync(LB_FULL, wincl, 31);
                    if (store_window(out.dst + pos, n, wincl - n, W)) {
                        Sink d;
                        d.dst = out.dst + pos + (wincl - n); d.n = 0; d.flags = 0; d.wr = true;
                        if (comma) d.put(',');
                        emit_scalar(d, &el, end);
                    }
                    pos += W;
                }
            }
        }
        u32 flags_all = cnt.flags;
        for (int d = 16; d > 0; d >>= 1) flags_all |= __shfl_xor_sync(LB_FULL, flags_all, d);
        out.flags |= flags_all;
        __syncwarp();
        if (out.dst) out.n = pos;
        else out.n += (u32)warp_sum((int)cnt.n);
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
    __shared__ JsonStage stg[4];
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
    Emitter e(t, di, s, lane, &tsm[(threadIdx.x >> 5) & 3], &stg[(threadIdx.x >> 5) & 3]);
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
