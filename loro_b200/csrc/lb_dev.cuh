// loro_b200 -- common device-side definitions (sm_90a).
//
// The same sources also compile under tests/emu/simt_emu.h (LB_SIMT_EMU) so that kernel logic can be
// exercised on a machine without a GPU; that build is test infrastructure and is never shipped.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "../../include/loro_b200.h"   // LB_MAX_NESTING: the stacks of every LoroValue walker

#ifdef LB_SIMT_EMU
#include "simt_emu.h"
#define LB_HD
#else
#include <cuda_runtime.h>
#define LB_HD __host__ __device__
// A launch that fails (no kernel image for this GPU, a bad configuration) fails the call: engine.cu records the error
// and throws LB_ERR_CUDA, so a library built for another architecture never returns empty results.
void lb_launch_failed(const char* kernel, cudaError_t e);
#define LB_LAUNCH(kernel, grid, block, smem, stream, ...)                  \
    do {                                                                   \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);        \
        cudaError_t lb_launch_e_ = cudaGetLastError();                     \
        if (lb_launch_e_ != cudaSuccess) lb_launch_failed(#kernel, lb_launch_e_); \
    } while (0)
#endif

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t i32;
typedef int64_t i64;

#define LB_FULL 0xffffffffu
// error tracing in the emulated test build only
#ifdef LB_SIMT_EMU
#define LB_ERR(x) (getenv("LB_EMU_TRACE") ? fprintf(stderr, "loro_b200(emu): %s at %s:%d\n", #x, __FILE__, __LINE__) : 0, (x))
#else
#define LB_ERR(x) (x)
#endif

// per-document codes (mirror include/loro_b200.h lb_doc_code)
enum { DOC_OK = 0, DOC_ERR_DECODE = 1, DOC_ERR_CHECKSUM = 2, DOC_ERR_MODE = 3, DOC_ERR_CORRUPT = 4,
       DOC_ERR_UNSUPPORTED = 5, DOC_ERR_CAPACITY = 6, DOC_ERR_FRONTIERS = 7 };

// value kinds of the `values` stream (reference: encoding/value.rs:39-161)
enum { VK_NULL = 0, VK_TRUE = 1, VK_FALSE = 2, VK_I64 = 3, VK_F64 = 4, VK_STR = 5, VK_BINARY = 6,
       VK_CONTAINER = 7, VK_DELETE_ONCE = 8, VK_DELETE_SEQ = 9, VK_DELTA_INT = 10, VK_LORO_VALUE = 11,
       VK_MARK_START = 12, VK_TREE_MOVE = 13, VK_LIST_MOVE = 14, VK_LIST_SET = 15, VK_RAW_TREE_MOVE = 16 };
// container types (reference: loro-common/src/lib.rs:293-347)
enum { CT_MAP = 0, CT_LIST = 1, CT_TEXT = 2, CT_TREE = 3, CT_MOVABLE = 4, CT_COUNTER = 5 };
// engine op classes
enum { OPK_SKIP = 0, OPK_SEQ_INS = 1, OPK_SEQ_DEL = 2, OPK_MAP_SET = 3, OPK_MAP_DEL = 4, OPK_UNSUPPORTED = 5, OPK_TREE = 6 };
// movable tree: parent slots that are not nodes (reference: state/tree_state.rs:69-77 TreeParentId)
#define TREE_ROOT 0xFFFFFFFFu
#define TREE_DELETED 0xFFFFFFFEu
#define TREE_UNEXIST 0xFFFFFFFDu
#define DELETED_ROOT_PEER 0xFFFFFFFFFFFFFFFFull   // loro-common/src/lib.rs:631 DELETED_TREE_ROOT
#define DELETED_ROOT_CTR 0x7FFFFFFF

#define PEER_NONE 0xFFFFu     // "no origin"
#define PEER_UNKNOWN 0xFFFEu  // the tracker's placeholder span (reference: tracker.rs:38-63)
#define UNKNOWN_LEN 0x3FFFFFFF  // u32::MAX / 4

// ------------------------------------------------------------------ byte cursor (bounds checked)
// Bytes are fetched eight at a time (one aligned 64-bit load per 8-byte window, validated by address so that code
// moving `p` directly stays correct): the decoders are bound by the latency of their byte loads, not by bandwidth.
// The batch byte buffer is padded, so the aligned window around any in-range byte is readable.
#define CUR_ERR_DEEP 2u   // Cur::err of a well-formed value that nests deeper than LB_MAX_NESTING (skip_loro_value_content)
struct Cur {
    const u8* p;
    const u8* end;
    u32 err;          // 0, 1 (malformed or past the end) or CUR_ERR_DEEP
    u64 buf;
    const u8* bp;   // address of the window held in buf (8-byte aligned), nullptr = none
    __device__ __forceinline__ Cur(const u8* b, size_t n) : p(b), end(b + n), err(0), buf(0), bp(nullptr) {}
    __device__ __forceinline__ size_t left() const { return (size_t)(end - p); }
    __device__ __forceinline__ bool empty() const { return p >= end; }
    __device__ __forceinline__ u8 get() {
        if (p >= end) { err = 1; return 0; }
        const u8* a = (const u8*)((uintptr_t)p & ~(uintptr_t)7);
        if (a != bp) { buf = *(const u64*)a; bp = a; }
        u8 v = (u8)(buf >> (8 * (unsigned)((uintptr_t)p & 7)));
        p++;
        return v;
    }
    __device__ __forceinline__ void skip(u64 n) {
        if (n > (u64)(end - p)) { err = 1; p = end; } else p += n;
    }
    // postcard varint == ULEB128 (reference: docs/encoding.md:869-946,1220-1239)
    __device__ __forceinline__ u64 varint() {
        u64 v = 0;
        int shift = 0;
        for (int i = 0; i < 10; i++) {
            u8 b = get();
            v |= (u64)(b & 0x7f) << shift;
            if (!(b & 0x80)) return v;
            shift += 7;
        }
        err = 1;
        return v;
    }
    // skips a varint of up to 19 bytes (i128 deltas), returning its low 64 bits
    __device__ __forceinline__ u64 varint_wide() {
        u64 v = 0;
        int shift = 0;
        for (int i = 0; i < 19; i++) {
            u8 b = get();
            if (shift < 64) v |= (u64)(b & 0x7f) << shift;
            if (!(b & 0x80)) return v;
            shift += 7;
        }
        err = 1;
        return v;
    }
    __device__ __forceinline__ i64 zigzag() {
        u64 v = varint();
        return (i64)(v >> 1) ^ -(i64)(v & 1);
    }
    // zigzag of an i128 delta truncated to i64 (column values are i32/u32/isize: the low 64 bits suffice
    // because accumulation is modular; reference: docs/encoding.md:1369-1395)
    __device__ __forceinline__ i64 zigzag_wide() {
        u64 v = varint_wide();
        return (i64)(v >> 1) ^ -(i64)(v & 1);
    }
    // SLEB128 (reference: docs/encoding.md:948-1054)
    __device__ __forceinline__ i64 sleb() {
        i64 result = 0;
        int shift = 0;
        u8 b;
        int n = 0;
        do {
            b = get();
            if (shift < 64) result |= (i64)((u64)(b & 0x7f) << shift);
            shift += 7;
            if (++n > 10) { err = 1; break; }
        } while (b & 0x80);
        if (shift < 64 && (b & 0x40)) result |= -((i64)1 << shift);
        return result;
    }
};

// ------------------------------------------------------------------ AnyRle column cursor
// reference: docs/encoding.md:1084-1115 ; moon/loro_codec/serde_columnar_any_rle.mbt
// value modes: 0 raw u8, 1 varint, 2 zigzag(i128) [DeltaRle deltas]
struct RleCur {
    Cur c;
    i64 run_left;   // >0: repeat `val`; <0: literals left
    i64 val;
    int mode;
    __device__ __forceinline__ RleCur(const u8* b, size_t n, int mode_) : c(b, n), run_left(0), val(0), mode(mode_) {}
    __device__ __forceinline__ i64 read_val() {
        if (mode == 0) return c.get();
        if (mode == 1) return (i64)c.varint();
        return c.zigzag_wide();
    }
    // returns false at end of column
    __device__ __forceinline__ bool next(i64* out) {
        if (run_left == 0) {
            if (c.empty()) return false;
            i64 sl = c.zigzag();
            if (sl == 0) { c.err = 1; return false; }
            if (sl > 0) { run_left = sl; val = read_val(); }
            else run_left = sl;
        }
        if (run_left > 0) { run_left--; *out = val; }
        else { run_left++; *out = read_val(); }
        return true;
    }
};

// ------------------------------------------------------------------ DeltaOfDelta bit cursor
// reference: docs/encoding.md:1126-1172 ; moon/loro_codec/serde_columnar_delta_of_delta_decode.mbt
struct DodCur {
    Cur* c;
    const u8* bits;
    size_t nbytes;
    size_t bitpos;
    i64 prev, delta;
    bool has_first;
    __device__ __forceinline__ void begin(Cur* cur) {
        c = cur;
        u8 tag = c->get();
        has_first = tag == 1;
        prev = 0;
        delta = 0;
        if (tag == 1) prev = c->zigzag();
        else if (tag != 0) c->err = 1;
        (void)c->get();  // last_used_bits: only needed by a whole-column decoder
        bits = c->p;
        nbytes = c->left();
        bitpos = 0;
    }
    __device__ __forceinline__ u32 bit() {
        if (bitpos >= nbytes * 8) { c->err = 1; return 0; }
        u32 v = (bits[bitpos >> 3] >> (7 - (bitpos & 7))) & 1;
        bitpos++;
        return v;
    }
    __device__ __forceinline__ u64 getbits(int n) {
        u64 v = 0;
        for (int i = 0; i < n; i++) v = (v << 1) | bit();
        return v;
    }
    // k-th value (k = 0 is the head)
    __device__ __forceinline__ i64 next(bool first) {
        if (first) {
            if (!has_first) c->err = 1;
            return prev;
        }
        i64 dod;
        if (!bit()) dod = 0;
        else if (!bit()) dod = (i64)getbits(7) - 63;
        else if (!bit()) dod = (i64)getbits(9) - 255;
        else if (!bit()) dod = (i64)getbits(12) - 2047;
        else if (!bit()) dod = (i64)getbits(21) - 1048575;
        else dod = (i64)getbits(64);
        delta += dod;
        prev += delta;
        return prev;
    }
    __device__ __forceinline__ void finish() { c->skip((bitpos + 7) / 8); }
};

// ------------------------------------------------------------------ warp helpers
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(LB_FULL, v, d);
        if (lane >= d) v += t;
    }
    return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(LB_FULL, v, d);
    return v;
}

// xxHash32 primes (reference: docs/encoding-xxhash32.md ; moon/loro_codec/xxhash32.mbt)
#define XXP1 0x9E3779B1u
#define XXP2 0x85EBCA77u
#define XXP3 0xC2B2AE3Du
#define XXP4 0x27D4EB2Fu
#define XXP5 0x165667B1u
#define XX_SEED_LORO 0x4F524F4Cu
__device__ __forceinline__ u32 rotl32(u32 x, int r) { return (x << r) | (x >> (32 - r)); }
