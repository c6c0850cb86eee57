// loro_b200 -- host orchestration + C ABI (include/loro_b200.h).
//
// The host side only sizes tables, launches kernels and copies results; every byte of decode / merge /
// materialisation work happens in the kernels of k_*.cuh.  There is no CPU fallback: with no CUDA device
// the entry points fail with LB_ERR_NO_DEVICE.
#include "../../include/loro_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>
#include <cstring>
#include <cstdio>
#include <cstdlib>
#include <sched.h>

#include "lb_defs.h"
#include "k_frame.cuh"
#include "k_decode.cuh"
#include "k_decode_warp.cuh"
#include "k_resolve.cuh"
#include "k_classify.cuh"
#include "k_checkout.cuh"
#include "k_seq.cuh"
#include "k_tree.cuh"
#include "k_state.cuh"
#include "k_export.cuh"
#include "k_json_updates.cuh"
#include "k_attr.cuh"
#include "k_cursor.cuh"
#include "host_stage.hpp"

static thread_local std::string g_last_error;
const char* lb_last_error(void) { return g_last_error.c_str(); }

#define CK(call)                                                                             \
    do {                                                                                     \
        cudaError_t e_ = (call);                                                             \
        if (e_ != cudaSuccess) {                                                             \
            g_last_error = std::string(#call) + ": " + cudaGetErrorString(e_);               \
            throw lb_status(LB_ERR_CUDA);                                                    \
        }                                                                                    \
    } while (0)

#ifndef LB_SIMT_EMU
void lb_launch_failed(const char* kernel, cudaError_t e) {
    g_last_error = std::string("launch of ") + kernel + ": " + cudaGetErrorString(e);
    throw lb_status(LB_ERR_CUDA);
}
#endif

// thread per doc helpers: the per-document sizes the host scans into table offsets ------------------
__global__ void k_doc_vv_cells(const DocInfo* __restrict__ docs, u32 n_docs, u32* __restrict__ vv_cells) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    vv_cells[d] = di.code == DOC_OK ? di.n_changes * di.P : 0;
}
__global__ void k_doc_atoms_mapslots(const DocInfo* __restrict__ docs, u32 n_docs, u32* __restrict__ atoms,
                                     u32* __restrict__ mapslots) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    bool ok = di.code == DOC_OK;
    atoms[d] = ok ? (u32)di.atom_total : 0;
    mapslots[d] = ok ? di.C * di.K : 0;
}
// tree node slots (k_tree.cuh) and, in *max_tree_atoms (zero on entry), the atoms of the largest tree document
__global__ void k_doc_tree_slots(const DocInfo* __restrict__ docs, u32 n_docs, u32* __restrict__ tree_slots,
                                 u32* __restrict__ max_tree_atoms) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    bool tree = di.code == DOC_OK && di.has_tree;
    tree_slots[d] = tree ? (u32)di.atom_total + di.C : 0;
    if (tree) atomicMax(max_tree_atoms, (u32)di.atom_total);
}
__global__ void k_pack_peers(const DocInfo* __restrict__ docs, u32 n_docs, const DocPeer* __restrict__ dpeer,
                             const u64* __restrict__ base, DocPeer* __restrict__ out) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    for (u32 p = 0; p < di.P; p++) out[base[d] + p] = dpeer[di.peer0 + p];
}
// multi-field scan: CTA f scans field f (offsets in bytes inside the strided records)
struct ScanJob { const u8* in; u8* out; size_t in_stride, out_stride; u64 n; };
struct ScanJobs { ScanJob j[8]; };
__global__ void k_excl_scan_multi(ScanJobs jobs) {
    const ScanJob& jb = jobs.j[blockIdx.x];
    const u8* in = jb.in; u8* out = jb.out; size_t in_stride = jb.in_stride, out_stride = jb.out_stride; u64 n = jb.n;
    __shared__ u64 warp_tot[32];
    __shared__ u64 carry_s;
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (u64 base = 0; base < n; base += blockDim.x) {
        u64 i = base + threadIdx.x;
        u64 v = i < n ? (u64) * (const u32*)(in + i * in_stride) : 0;
        u64 s = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            u64 t = __shfl_up_sync(LB_FULL, s, d);
            if (lane >= d) s += t;
        }
        if (lane == 31) warp_tot[w] = s;
        __syncthreads();
        if (w == 0) {
            u64 t = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : 0;
            u64 ts = t;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                u64 u = __shfl_up_sync(LB_FULL, ts, d);
                if (lane >= d) ts += u;
            }
            warp_tot[lane] = ts - t;
        }
        __syncthreads();
        u64 carry = carry_s;
        if (i < n) *(u64*)(out + i * out_stride) = carry + warp_tot[w] + s - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_s = carry + warp_tot[w] + s;
        __syncthreads();
    }
    if (threadIdx.x == 0) *(u64*)(out + n * out_stride) = carry_s;
}

// warp per segment: copy blobs between device buffers (lb_docset: the stored state of a document enters the next batch,
// the re-exported blobs leave the batch).  Sources and destinations are 16-byte aligned.
struct CopySeg { const u8* src; u8* dst; u64 len; };
__global__ void k_copy_segments(const CopySeg* __restrict__ segs, u32 n) {
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (w >= n) return;
    CopySeg sg = segs[w];
    u64 n16 = sg.len >> 4;
    const uint4* s4 = (const uint4*)sg.src;
    uint4* d4 = (uint4*)sg.dst;
    for (u64 i = lane; i < n16; i += 32) d4[i] = s4[i];
    for (u64 i = (n16 << 4) + lane; i < sg.len; i += 32) sg.dst[i] = sg.src[i];
}

namespace {

// LB_PHASE_TRACE: diagnostics on stderr.  Read at every use, so that a process can switch it on between batches.
inline bool phase_trace() { return getenv("LB_PHASE_TRACE") != nullptr; }

// Device blocks that lived until their batch was freed are kept per device, by size class, and handed to the next batch
// that asks for the same class: a service imports batch after batch of similar shape, and the stream-ordered pool took
// up to hundreds of milliseconds (host-blocking) to find or map room for the multi-GB row tables of a step -- 68 ms per
// step on config C5.  Blocks a batch gives back early (Dev::release) still go to the pool, so their memory stays
// available to every later size.  lb_device_trim() empties the cache.
struct BlockCache {
    std::mutex mu;
    std::unordered_map<size_t, std::vector<void*>> free_;
    size_t bytes = 0;
};
BlockCache& block_cache(int device) {
    static BlockCache caches[64];
    return caches[(unsigned)device % 64];
}
size_t cache_cap_bytes() {   // LB_DEV_CACHE_GB, default 85 % of the device's memory
    static const size_t cap = [] {
        const char* e = getenv("LB_DEV_CACHE_GB");
        if (e) return (size_t)(atof(e) * 1e9);
        size_t fr = 0, tot = 0;
        if (cudaMemGetInfo(&fr, &tot) != cudaSuccess) tot = (size_t)64e9;
        return (size_t)((double)tot * 0.85);
    }();
    return cap;
}
inline size_t size_class(size_t sz) {   // 8 classes per power of two (at most 12.5 % above the request), 256-byte granules
    sz = (sz + 255) & ~(size_t)255;
#ifndef LB_SIMT_EMU
    if (sz > 4096) {
        int e = 63 - __builtin_clzll((unsigned long long)(sz - 1));
        size_t step = (size_t)1 << (e - 3);
        sz = (sz + step - 1) & ~(step - 1);
    }
#endif
    return sz;
}
void cache_flush(int device, cudaStream_t st) {
    BlockCache& bc = block_cache(device);
    std::lock_guard<std::mutex> g(bc.mu);
    for (auto& kv : bc.free_) for (void* p : kv.second) cudaFreeAsync(p, st);
    bc.free_.clear();
    bc.bytes = 0;
}

// Batch streams are recycled per device: memory a batch frees early goes back to the stream-ordered pool, and the pool
// serves a later request fastest when it comes from the stream the memory was freed on.
struct StreamCache {
    std::mutex mu;
    std::vector<cudaStream_t> idle;
};
StreamCache& stream_cache(int device) {
    static StreamCache caches[64];
    return caches[(unsigned)device % 64];
}
cudaStream_t stream_take(int device) {
    StreamCache& sc = stream_cache(device);
    {
        std::lock_guard<std::mutex> g(sc.mu);
        if (!sc.idle.empty()) { cudaStream_t s = sc.idle.back(); sc.idle.pop_back(); return s; }
    }
    cudaStream_t s = nullptr;
    if (cudaStreamCreate(&s) != cudaSuccess) return nullptr;
    return s;
}
void stream_give(int device, cudaStream_t s) {
    StreamCache& sc = stream_cache(device);
    std::lock_guard<std::mutex> g(sc.mu);
    if (sc.idle.size() < 4 && !getenv("LB_NO_STREAM_REUSE")) sc.idle.push_back(s);
    else cudaStreamDestroy(s);
}

struct Dev {  // owns every device allocation of a batch
    cudaStream_t stream = nullptr;
    int device = 0;
    std::vector<std::pair<void*, size_t>> ptrs;   // whole blocks in use
    // Blocks the batch is done with before it ends (the tracker pools after phase 5) stay with the batch: later tables
    // are carved out of them (same stream, so the order of use is the order of enqueueing) and at the end they go to
    // the block cache whole.  Handing them to the stream-ordered pool and asking it for the export tables made the
    // multi-GB requests block the host at random (0.3 ms on one step, 120 ms -- once 1.2 s -- on the next).
    struct Carve { size_t off, need; bool live; };
    struct Region { char* base; size_t size, used; std::vector<Carve> stack; };
    std::vector<Region> released;
    size_t bytes = 0;
    double alloc_ms = 0;   // host time inside the allocator (it blocks when the pool has to map memory)
    template <class T>
    T* alloc(size_t n, bool zero = false) {
        void* p = nullptr;
        const size_t want = (n ? n : 1) * sizeof(T);
        const size_t sz = size_class(want);
        auto t0 = std::chrono::steady_clock::now();
        bool carved = false;
#ifndef LB_SIMT_EMU
        {
            const size_t need = (want + 255) & ~(size_t)255;
            for (auto& r : released)
                if (r.size - r.used >= need) { p = r.base + r.used; r.stack.push_back(Carve{r.used, need, true}); r.used += need; carved = true; break; }
        }
        if (!p) {
            BlockCache& bc = block_cache(device);
            std::lock_guard<std::mutex> g(bc.mu);
            auto it = bc.free_.find(sz);
            if (it != bc.free_.end() && !it->second.empty()) { p = it->second.back(); it->second.pop_back(); bc.bytes -= sz; }
        }
#endif
        if (!p) {
            cudaError_t e = cudaMallocAsync(&p, sz, stream);
            if (e != cudaSuccess) {   // out of memory with blocks parked in the cache: give them back and try once more
                cudaGetLastError();
                cache_flush(device, stream);
                cudaStreamSynchronize(stream);
                e = cudaMallocAsync(&p, sz, stream);
            }
            if (e != cudaSuccess) {
                g_last_error = std::string("cudaMallocAsync(") + std::to_string(sz) + "): " + cudaGetErrorString(e);
                throw lb_status(LB_ERR_OOM);
            }
        }
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        alloc_ms += ms;
        if (ms > 1.0 && phase_trace()) fprintf(stderr, "[trace] slow alloc: %zu bytes took %.3f ms\n", sz, ms);
        if (!carved) { ptrs.push_back({p, sz}); bytes += sz; }
        if (zero) CK(cudaMemsetAsync(p, 0, want, stream));
        return (T*)p;
    }
    // the batch has enqueued the last consumer of a table: its block becomes room for later tables (see `released`)
    template <class T>
    void release(T*& p) {
        if (!p) return;
        for (size_t i = 0; i < ptrs.size(); i++)
            if (ptrs[i].first == (void*)p) {
#ifndef LB_SIMT_EMU
                released.push_back(Region{(char*)p, ptrs[i].second, 0, {}});
#else
                cudaFreeAsync((void*)p, stream);
#endif
                ptrs[i] = ptrs.back();
                ptrs.pop_back();
                break;
            }
        // a table carved out of a released block: its room is reusable once everything carved after it is gone too
        for (auto& r : released) {
            if ((char*)p < r.base || (char*)p >= r.base + r.size) continue;
            const size_t off = (size_t)((char*)p - r.base);
            for (auto& c : r.stack) if (c.off == off) c.live = false;
            while (!r.stack.empty() && !r.stack.back().live) { r.used = r.stack.back().off; r.stack.pop_back(); }
            break;
        }
        p = nullptr;
    }
    // the batch is gone and its stream has been synchronised: the blocks are free for any stream
    void free_all() {
#ifndef LB_SIMT_EMU
        for (auto& r : released) ptrs.push_back({(void*)r.base, r.size});
        released.clear();
        BlockCache& bc = block_cache(device);
        std::lock_guard<std::mutex> g(bc.mu);
        for (auto& pr : ptrs) {
            if (bc.bytes + pr.second <= cache_cap_bytes()) { bc.free_[pr.second].push_back(pr.first); bc.bytes += pr.second; }
            else cudaFreeAsync(pr.first, stream);
        }
#else
        for (auto& pr : ptrs) cudaFreeAsync(pr.first, stream);
#endif
        ptrs.clear();
    }
};

}  // namespace

// Events on the batch stream, in pipeline order: EV_x is recorded when phase x has been enqueued (mark), and a phase's
// device time is the interval from the event before it (timings_from_events).
enum BatchEvent { EV_START, EV_H2D, EV_FRAME, EV_DECODE, EV_RESOLVE, EV_CLASSIFY, EV_INTEGRATE, EV_CURSORS, EV_TREE, EV_MATERIALISE,
                  EV_ATTRIBUTION, EV_EXPORT, EV_D2H, EV_COUNT };

// The sizes of the batch-wide tables, each read back from the device by the phase that scans it; the later phases, the
// on-demand exports, the counters and the debug tables are sized by them.
struct BatchSizes {
    u64 blocks = 0;                                                            // frame
    u64 peers = 0, keys = 0, cids = 0, changes = 0, deps = 0, rows = 0, dels = 0, pos = 0, pos_bytes = 0, tree_ops = 0;  // decode
    u64 atoms = 0, map_slots = 0;                                              // resolve
    u64 leaves = 0, nodes = 0, runs = 0, cvv = 0;                              // classify: the sequence trackers' pools
};

// A per-document result that comes home whole on the first accessor call: the device buffer, its bytes, and the host
// copy (from lbstage::host_cache, zero-terminated) once fetched.
struct HostResult {
    u8* d = nullptr; u64 total = 0; char* host = nullptr; bool fetched = false;
    lb_status fetch(cudaStream_t st, const char* failed) {
        if (fetched) return LB_OK;
        if (!host) host = (char*)lbstage::host_cache().take(total + 1);
        if (!host) { g_last_error = "out of host memory"; return LB_ERR_OOM; }
        if (total && !lbstage::download(d, (u8*)host, total, st)) { g_last_error = failed; return LB_ERR_CUDA; }
        host[total] = 0;
        fetched = true;
        return LB_OK;
    }
};

struct lb_batch {
    Dev dev;
    size_t n_docs = 0;
    uint32_t flags = 0;
    bool owns_bytes = false;
    // device state
    BatchTables tb{};             // every batch-wide table (the input bytes at tb.bytes), kept for export(updates(from))
    u64* d_offs = nullptr;
    u32* d_lens = nullptr;
    size_t n_blobs = 0;                       // blobs in the byte buffer (>= n_docs: import_batch groups)
    std::vector<u32> blob_doc, doc_blob0;     // blob -> document ; document -> first blob (n_docs + 1)
    std::vector<u32> doc_nprior;              // lb_docset_import: leading blobs of each document that restate its earlier state
    // checkout requests (k_checkout.cuh), empty when the batch has none: document d is built at the ids
    // [ck_range[2d], ck_range[2d + 1]) of ck_peer / ck_ctr, or at the latest version when ck_range[2d] == CK_LATEST
    std::vector<u32> ck_range;
    std::vector<u64> ck_peer;
    std::vector<i32> ck_ctr;
    bool stored_only = false;                 // lb_docset_checkout / lb_docset_read: nothing was imported, the status spans
                                              // stay empty
    DocInfo* d_docs = nullptr;
    BatchSizes n;
    // per-document results; document d's part is placed by docs[d].json_off / json_len, by [attr_off[d],
    // attr_off[d + 1]) (LB_FLAG_ATTRIBUTION, k_attr.cuh; the offsets come home with the text) and by xdocs[d].exp_off /
    // exp_len (phase 7: one FastUpdates blob per document)
    HostResult json, attr, exported;
    u64* d_attr_off = nullptr;
    std::vector<u64> attr_off;
    // LB_FLAG_CURSORS (k_cursor.cuh): every Text / List rope in document order and by id, for lb_batch_cursor_pos
    CursorTables cur{};
    std::vector<XDoc> xdocs;
    std::unordered_map<size_t, std::vector<uint8_t>> from_exports;   // last lb_doc_export_updates(from) per document
    std::mutex export_mu;                     // on-demand exports of one batch run one at a time
    u64 n_segs = 0, fc_cap = 0;   // phase 7: segments (changes + extra segments of split ones), fc_* table capacity
    // host results
    std::vector<DocInfo> docs;
    std::vector<DocPeer> dpeer;          // packed: document d owns [peer_base[d], peer_base[d] + P)
    std::vector<u64> peer_base;
    // host-buffer entry point: the JSON goes home on a second stream while the export phase still computes
    bool eager_json = false, json_ok = true;
    cudaStream_t stream2 = nullptr;
    cudaEvent_t json_ev = nullptr;
    std::thread json_thread;
    std::vector<lb_id_span> spans[4];          // success, pending, vv, frontiers of all documents, flat
    std::vector<size_t> span_off[4];           // document d owns [span_off[k][d], span_off[k][d + 1])
    std::vector<uint64_t> doc_ids;
    lb_counters counters{};
    lb_timings timings{};
    std::chrono::steady_clock::time_point t_call = std::chrono::steady_clock::now(), t_tail = t_call;
    cudaEvent_t ev[EV_COUNT];
    bool ev_recorded[EV_COUNT] = {};
    bool ev_created = false;
};

// Persistent documents (lb_docset_*): what a document keeps between imports is its change store in wire form -- the
// FastUpdates blob it would export (ExportMode::all_updates), resident in device memory -- exactly what the reference's
// ChangeStore keeps (encoded blocks in a kv store, change_store.rs:60-110).  A document that still has pending changes
// keeps the blobs it was built from instead (pending changes are not part of an export).
struct DocsetBuf {     // one device buffer per import generation, shared by the documents stored in it
    u8* d = nullptr;
    size_t bytes = 0;
    ~DocsetBuf() { if (d) cudaFree(d); }
};
struct DocsetBlob { std::shared_ptr<DocsetBuf> buf; u64 off; u32 len; };
struct DocsetDoc { std::vector<DocsetBlob> blobs; };
struct lb_docset {
    int device = 0;
    std::mutex mu;
    std::unordered_map<u64, DocsetDoc> docs;
    u64 stored_bytes = 0;
};

// The answers of one lb_batch_export_updates call, in host memory that outlives the batch.
struct lb_exports {
    struct Answer { lb_status status; const char* error; const uint8_t* bytes; size_t len; };
    std::vector<Answer> answers;                        // one per request
    std::vector<std::unique_ptr<uint8_t[]>> bufs;       // the packed blobs of each round, and the all_updates copies
};

namespace {

const int TPB = 128;
inline unsigned nblk(u64 n, int tpb = TPB) { return (unsigned)((n + tpb - 1) / tpb); }

// Every kernel a batch launches goes through here: on the batch's stream, and counted in lb_timings.kernel_launches.
#define LB_BATCH_LAUNCH(b, kernel, grid, block, smem, ...)                          \
    do {                                                                            \
        LB_LAUNCH(kernel, grid, block, smem, (b)->dev.stream, __VA_ARGS__);         \
        (b)->timings.kernel_launches++;                                             \
    } while (0)

// the u32 segment and final-change tables of phase 7, for its allocation and the growth paths
u32* BatchTables::* const SG_TABLES[] = {
    &BatchTables::sg_src, &BatchTables::sg_r0, &BatchTables::sg_from, &BatchTables::sg_atoms, &BatchTables::sg_est,
    &BatchTables::sg_nmops, &BatchTables::sg_ndel, &BatchTables::sg_nrows, &BatchTables::sg_last_head, &BatchTables::sg_skip};
u32* BatchTables::* const FC_TABLES[] = {
    &BatchTables::fc_src, &BatchTables::fc_pos, &BatchTables::fc_r0, &BatchTables::fc_from, &BatchTables::fc_atoms,
    &BatchTables::fc_nrows, &BatchTables::fc_ndel, &BatchTables::fc_skip, &BatchTables::fc_tail, &BatchTables::fc_est};

// the export encoder over NOB output blocks (retry = 1: only the blocks that outgrew their staging slot, into their
// retry slots), in the build that is faster for that many (k_export.cuh); cuts: some change is cut at the end of its span
void launch_exp_encode(lb_batch* b, u64 NOB, const BatchTables& xt, XBlock* xb, u32* xscratch, u8* out, int retry, bool cuts) {
    if (!NOB) return;
    const bool capped = NOB >= LB_XENC_BOUNDED_MIN_BLOCKS;
    if (cuts && capped) LB_BATCH_LAUNCH(b, k_exp_encode_cut<1>, nblk(NOB, 64), 64, 0, b->d_docs, NOB, xt, xb, xscratch, out, retry);
    else if (cuts) LB_BATCH_LAUNCH(b, k_exp_encode_cut<0>, nblk(NOB, 64), 64, 0, b->d_docs, NOB, xt, xb, xscratch, out, retry);
    else if (capped) LB_BATCH_LAUNCH(b, k_exp_encode<1>, nblk(NOB, 64), 64, 0, b->d_docs, NOB, xt, xb, xscratch, out, retry);
    else LB_BATCH_LAUNCH(b, k_exp_encode<0>, nblk(NOB, 64), 64, 0, b->d_docs, NOB, xt, xb, xscratch, out, retry);
}

// CTAs of k_seq_integrate that the device holds at once, computed once per device: a batch that needs more gets that
// many, whose warps take documents from a queue until none are left.  The emulated build has no occupancy query: one
// CTA, so that its tests pass many documents through each warp.
unsigned seq_resident_ctas(int device) {
#ifdef LB_SIMT_EMU
    (void)device;
    return 1;
#else
    static std::atomic<unsigned> ctas[64];
    std::atomic<unsigned>& n = ctas[(unsigned)device % 64];
    if (!n.load(std::memory_order_relaxed)) {
        int per_sm = 0, sms = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_seq_integrate<1>, 32 * LB_SEQ_WARPS, 0));
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        if (per_sm < 1 || sms < 1) {
            g_last_error = "k_seq_integrate: no CTA fits a multiprocessor";
            throw lb_status(LB_ERR_CUDA);
        }
        n.store((unsigned)per_sm * (unsigned)sms, std::memory_order_relaxed);
    }
    return n.load(std::memory_order_relaxed);
#endif
}

void mark(lb_batch* b, BatchEvent e) {
    CK(cudaEventRecord(b->ev[e], b->dev.stream));
    b->ev_recorded[e] = true;
}

template <class T>
T d2h_one(lb_batch* b, const T* src) {
    T v;
    CK(cudaMemcpyAsync(&v, src, sizeof(T), cudaMemcpyDeviceToHost, b->dev.stream));
    CK(cudaStreamSynchronize(b->dev.stream));
    return v;
}

// LB_PHASE_TRACE=1: host wall clock between named points (each one synchronises the stream: diagnosis only)
void trace_point(lb_batch* b, const char* name) {
    if (!phase_trace()) return;
    static std::chrono::steady_clock::time_point last = std::chrono::steady_clock::now();
    cudaStreamSynchronize(b->dev.stream);
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[trace] %-24s %8.3f ms\n", name, std::chrono::duration<double, std::milli>(now - last).count());
    last = now;
}

void run_scans(lb_batch* b, std::vector<ScanJob> jobs) {
    for (size_t i = 0; i < jobs.size(); i += 8) {
        ScanJobs sj;
        memset(&sj, 0, sizeof(sj));
        unsigned n = 0;
        for (; n < 8 && i + n < jobs.size(); n++) sj.j[n] = jobs[i + n];
        LB_BATCH_LAUNCH(b, k_excl_scan_multi, n, 1024, 0, sj);
    }
}
// The jobs of run_scans: n u32 counts summed exclusively into u64 offsets, the total at index n.  The offsets are the
// member `field` of the records `rec`, or a plain array; the counts a plain array, or the member `count` of the same
// records.  The byte offsets and strides of the job follow from the member pointers.
template <class T>
ScanJob scan_job(const u32* counts, T* rec, u64 T::*field, u64 n) { return ScanJob{(const u8*)counts, (u8*)&(rec->*field), 4, sizeof(T), n}; }
template <class T>
ScanJob scan_job(T* rec, u32 T::*count, u64 T::*field, u64 n) { return ScanJob{(const u8*)&(rec->*count), (u8*)&(rec->*field), sizeof(T), sizeof(T), n}; }
ScanJob scan_job(const u32* counts, u64* offsets, u64 n) { return ScanJob{(const u8*)counts, (u8*)offsets, 4, 8, n}; }

// Phase 7's final-change tables (FC_TABLES and fc_block) with room for `cap` slots: reallocated, zeroed, when they hold
// fewer.  What they held is not kept: each export pass fills them afresh.
void grow_fc_tables(lb_batch* b, u64 cap) {
    if (cap <= b->fc_cap) return;
    Dev& dv = b->dev;
    b->fc_cap = cap;
    for (auto m : FC_TABLES) { dv.release(b->tb.*m); b->tb.*m = dv.alloc<u32>(cap, true); }
    dv.release(b->tb.fc_block);
    b->tb.fc_block = dv.alloc<u8>(cap);
}

// The encode end of phase 7, after the stores (k_exp_store) have cut every document's changes into output blocks;
// shared by the batch's export and export_from.  Block list with scratch and staging slots, one encode into the slots,
// layout (the lengths are exact, so are the offsets and the retry slots), the encode again of the blocks that outgrew
// their slot, into retry slots of their exact size (only when there are any: the retry bytes come back with the blob
// sizes), then the blobs assembled per document.
// cuts: some span of the pass ends inside a change (the encoder build that honours fc_tail).
// Returns the export buffer (*total bytes, document d's blob at xt.xdoc[d].exp_off).
u8* export_encode(lb_batch* b, const BatchTables& xt, u64* total, bool cuts) {
    Dev& dv = b->dev;
    const u32 D = (u32)b->n_docs;
    u32* cnt = dv.alloc<u32>(3 * (u64)(D + 1));
    u32 *n_a = cnt, *n_b = cnt + (D + 1), *n_c = cnt + 2 * (D + 1);
    LB_BATCH_LAUNCH(b, k_exp_sizes, nblk(D), TPB, 0, b->d_docs, D, xt, n_a, n_b, n_c);
    run_scans(b, {scan_job(n_a, xt.xdoc, &XDoc::ob0, D), scan_job(n_b, xt.xdoc, &XDoc::scratch0, D),
                  scan_job(n_c, xt.xdoc, &XDoc::stage0, D)});
    XDoc xtot = d2h_one(b, xt.xdoc + D);
    const u64 NOB = xtot.ob0, NSCR = xtot.scratch0, NSTG = xtot.stage0;
    XBlock* xb = dv.alloc<XBlock>(NOB + 1);
    u32* xscratch = dv.alloc<u32>(NSCR + 1);
    u8* xstage = dv.alloc<u8>(NSTG + 16);
    const char* cap_env = getenv("LB_EXPORT_STAGE_CAP");   // testing hook: smaller slots send blocks through the retry
    const u32 stage_max = cap_env ? (u32)strtoul(cap_env, nullptr, 10) : 0xFFFFFFFFu;
    trace_point(b, "store+sizes");
    LB_BATCH_LAUNCH(b, k_exp_list, nblk(D), TPB, 0, b->d_docs, D, xt, xb, stage_max);
    launch_exp_encode(b, NOB, xt, xb, xscratch, xstage, 0, cuts);
    LB_BATCH_LAUNCH(b, k_exp_layout, nblk(D), TPB, 0, b->d_docs, D, xt, xb, n_a, n_b, n_c);
    trace_point(b, "encode");
    run_scans(b, {scan_job(n_a, xt.xdoc, &XDoc::exp_off, D), scan_job(n_b, xt.xdoc, &XDoc::ovf0, D),
                  scan_job(n_c, xt.xdoc, &XDoc::restage0, D)});
    xtot = d2h_one(b, xt.xdoc + D);
    const u64 XT = xtot.exp_off, NOVF = xtot.ovf0, NRST = xtot.restage0;
    if (phase_trace())
        fprintf(stderr, "[trace] export: %llu blocks, %llu outgrew their staging slot; %llu staging bytes for %llu exported\n",
                (unsigned long long)NOB, (unsigned long long)NOVF, (unsigned long long)NSTG, (unsigned long long)XT);
    trace_point(b, "layout scan + size d2h");
    u8* out = dv.alloc<u8>(XT + 16, true);
    trace_point(b, "export buffer alloc+zero");
    u8* xrestage = nullptr;
    if (NOVF) {
        xrestage = dv.alloc<u8>(NRST + 16);
        launch_exp_encode(b, NOB, xt, xb, xscratch, xrestage, 1, cuts);
    }
    LB_BATCH_LAUNCH(b, k_exp_finish, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, xt, xb, xstage, xrestage, out);
    trace_point(b, "assemble");
    dv.release(cnt); dv.release(xb); dv.release(xscratch); dv.release(xstage); dv.release(xrestage);
    *total = XT;
    return out;
}

// The device tables of the import pipeline that one phase makes and a later one reads, besides BatchTables.
struct PhaseLinks {
    u32* doc_blob0 = nullptr;                                                  // frame -> resolve
    uint2* ck_range = nullptr; u64* ck_peer = nullptr; i32* ck_ctr = nullptr;  // checkout requests: frame -> resolve
    unsigned long long* acc = nullptr;                                         // state hash and counts: materialise -> results
};

const u32 SEQ_LEAF_W = 32;   // slots per leaf of the sequence trackers = lanes per warp (k_seq.cuh)

// phase 1: the blobs' blocks, and each document's block range
void phase_frame(lb_batch* b, PhaseLinks& ln) {
    Dev& dv = b->dev; cudaStream_t st = dv.stream; BatchTables& t = b->tb; const u32 D = (u32)b->n_docs, Q = (u32)b->n_blobs;
    b->d_docs = dv.alloc<DocInfo>(D + 1, true);
    u32* d_blob_code = dv.alloc<u32>(Q + 1, true);
    u32* d_blob_nblocks = dv.alloc<u32>(Q + 1, true);
    u64* d_blob_block0 = dv.alloc<u64>(Q + 2, true);
    u32* d_blob_doc = dv.alloc<u32>(Q + 1);
    ln.doc_blob0 = dv.alloc<u32>(D + 2);
    CK(cudaMemcpyAsync(d_blob_doc, b->blob_doc.data(), sizeof(u32) * Q, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ln.doc_blob0, b->doc_blob0.data(), sizeof(u32) * (D + 1), cudaMemcpyHostToDevice, st));
    LB_BATCH_LAUNCH(b, k_frame_count, nblk((u64)Q * 32, 128), 128, 0, t.bytes, b->d_offs, b->d_lens, Q, d_blob_code, d_blob_nblocks);
    run_scans(b, {scan_job(d_blob_nblocks, d_blob_block0, Q)});
    u32* d_doc_nprior = nullptr;
    if (!b->doc_nprior.empty()) {
        d_doc_nprior = dv.alloc<u32>(D + 1);
        CK(cudaMemcpyAsync(d_doc_nprior, b->doc_nprior.data(), sizeof(u32) * D, cudaMemcpyHostToDevice, st));
    }
    if (!b->ck_range.empty()) {   // the host vectors live as long as the batch: no synchronise needed
        const size_t NF = b->ck_peer.size();
        ln.ck_range = dv.alloc<uint2>(D);
        ln.ck_peer = dv.alloc<u64>(NF);
        ln.ck_ctr = dv.alloc<i32>(NF);
        CK(cudaMemcpyAsync(ln.ck_range, b->ck_range.data(), sizeof(u32) * 2 * D, cudaMemcpyHostToDevice, st));
        if (NF) {
            CK(cudaMemcpyAsync(ln.ck_peer, b->ck_peer.data(), sizeof(u64) * NF, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(ln.ck_ctr, b->ck_ctr.data(), sizeof(i32) * NF, cudaMemcpyHostToDevice, st));
        }
    }
    LB_BATCH_LAUNCH(b, k_frame_docs, nblk(D), TPB, 0, D, ln.doc_blob0, d_blob_code, d_blob_block0, d_doc_nprior, b->d_docs);
    b->n.blocks = d2h_one(b, d_blob_block0 + Q);
    t.blocks = dv.alloc<BlockInfo>(b->n.blocks + 1, true);
    LB_BATCH_LAUNCH(b, k_frame_fill, nblk(Q), TPB, 0, t.bytes, b->d_offs, b->d_lens, Q, d_blob_doc, d_blob_code, d_blob_block0, ln.doc_blob0, t.blocks);
    mark(b, EV_FRAME);
}

// phase 2: the blocks' column sizes, scanned into the batch-wide tables, then the columns decoded into them
void phase_decode(lb_batch* b) {
    Dev& dv = b->dev; BatchTables& t = b->tb;
    BlockInfo* blk = t.blocks;
    const u64 B = b->n.blocks;
    if (B) LB_BATCH_LAUNCH(b, k_block_count, nblk(B, 64), 64, 0, t.bytes, blk, B);
    run_scans(b, {scan_job(blk, &BlockInfo::n_peers, &BlockInfo::peer0, B), scan_job(blk, &BlockInfo::n_keys, &BlockInfo::key0, B),
                  scan_job(blk, &BlockInfo::n_cids, &BlockInfo::cid0, B), scan_job(blk, &BlockInfo::n_changes, &BlockInfo::ch0, B),
                  scan_job(blk, &BlockInfo::n_deps, &BlockInfo::dep0, B), scan_job(blk, &BlockInfo::n_ops, &BlockInfo::op0, B),
                  scan_job(blk, &BlockInfo::n_dels, &BlockInfo::del0, B), scan_job(blk, &BlockInfo::n_pos, &BlockInfo::pos0, B),
                  scan_job(blk, &BlockInfo::pos_bytes, &BlockInfo::posb0, B), scan_job(blk, &BlockInfo::n_tree, &BlockInfo::tr0, B)});
    BlockInfo tot = d2h_one(b, blk + B);
    u64 NP = tot.peer0, NK = tot.key0, NC = tot.cid0, NCH = tot.ch0, ND = tot.dep0, NR = tot.op0, NDEL = tot.del0;
    u64 NPOS = tot.pos0, NPOSB = tot.posb0, NTR = tot.tr0;
    if (NTR >= 0xFFFFFFFFull || NPOS >= 0xFFFFFFFFull) { g_last_error = "batch too large: tree ops / positions must fit 32 bits"; throw lb_status(LB_ERR_INVALID_ARG); }
    if (NR >= 0xFFFFFFFFull || NCH >= 0xFFFFFFFFull) { g_last_error = "batch too large: op rows / changes must fit 32 bits"; throw lb_status(LB_ERR_INVALID_ARG); }
    b->n = BatchSizes{B, NP, NK, NC, NCH, ND, NR, NDEL, NPOS, NPOSB, NTR};
    t.peer_id = dv.alloc<u64>(NP);
    t.key_off = dv.alloc<u64>(NK); t.key_len = dv.alloc<u32>(NK);
    t.cid_root = dv.alloc<u8>(NC); t.cid_type = dv.alloc<u8>(NC); t.cid_peer_idx = dv.alloc<u32>(NC); t.cid_koc = dv.alloc<i32>(NC);
    t.ch_block = dv.alloc<u32>(NCH); t.ch_counter = dv.alloc<i32>(NCH); t.ch_len = dv.alloc<u32>(NCH);
    t.ch_lamport_wire = dv.alloc<u32>(NCH); t.ch_ts = dv.alloc<i64>(NCH); t.ch_dep0 = dv.alloc<u64>(NCH);
    t.ch_msg_off = dv.alloc<u64>(NCH); t.ch_msg_len = dv.alloc<u32>(NCH, true);
    t.ch_ndeps = dv.alloc<u32>(NCH); t.ch_dep_self = dv.alloc<u8>(NCH); t.ch_op0 = dv.alloc<u64>(NCH);
    t.ch_nops = dv.alloc<u32>(NCH, true);
    t.dep_peer_idx = dv.alloc<u32>(ND); t.dep_counter = dv.alloc<i32>(ND);
    t.op_cid = dv.alloc<u32>(NR); t.op_prop = dv.alloc<i32>(NR); t.op_vtype = dv.alloc<u8>(NR); t.op_len = dv.alloc<u32>(NR);
    t.op_counter = dv.alloc<i32>(NR); t.op_change = dv.alloc<u32>(NR); t.op_val_off = dv.alloc<u64>(NR);
    t.op_val_len = dv.alloc<u32>(NR); t.op_del = dv.alloc<u32>(NR);
    t.del_peer_idx = dv.alloc<u32>(NDEL); t.del_counter = dv.alloc<i32>(NDEL); t.del_len = dv.alloc<i32>(NDEL);
    t.pos_off = dv.alloc<u64>(NPOS); t.pos_len = dv.alloc<u32>(NPOS); t.pos_pool = dv.alloc<u8>(NPOSB + 8);
    t.tr_target_peer = dv.alloc<u32>(NTR); t.tr_target_ctr = dv.alloc<i32>(NTR); t.tr_parent_kind = dv.alloc<u8>(NTR);
    t.tr_parent_peer = dv.alloc<u32>(NTR); t.tr_parent_ctr = dv.alloc<i32>(NTR); t.tr_pos = dv.alloc<u32>(NTR);
    t.dw_stats = dv.alloc<unsigned long long>(4, true);
    if (B) {
        // block decoder (DESIGN.md section 4): LB_DECODE=warp selects a warp per block on TMA-staged shared memory
        // (k_decode_warp.cuh); anything else, or nothing, a thread per block one column at a time (k_decode.cuh)
        static const char* mode_env = getenv("LB_DECODE");
        static const bool warp = mode_env && !strcmp(mode_env, "warp");
        if (!warp) LB_BATCH_LAUNCH(b, k_block_decode_cols, nblk(B, 64), 64, 0, t.bytes, blk, B, t);
        else {
            const size_t smem = sizeof(DwWarp) * DW_WARPS;
#ifndef LB_SIMT_EMU
            static bool attr_set = false;
            if (!attr_set) { CK(cudaFuncSetAttribute(k_block_decode_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr_set = true; }
#endif
            LB_BATCH_LAUNCH(b, k_block_decode_warp, nblk(B, DW_WARPS), 32 * DW_WARPS, smem, t.bytes, blk, B, t);
        }
    }
    mark(b, EV_DECODE);
    // SURVEY 8d algorithmic bytes of decode: blob bytes read + SoA written
    b->timings.decode_bytes_written = NR * 13 + NCH * (4 + 4 + 8 + 4) + ND * 12;
}

// phase 3: each document's peers, containers and keys, causal order, version vectors and frontiers (and, for a
// checkout, where each peer's history ends), then its atom and map-slot bases
void phase_resolve(lb_batch* b, const PhaseLinks& ln) {
    Dev& dv = b->dev; BatchTables& t = b->tb; BatchSizes& n = b->n; const u32 D = (u32)b->n_docs;
    const u64 NP = n.peers, NC = n.cids, NK = n.keys, NCH = n.changes;
    t.dpeer = dv.alloc<DocPeer>(NP, true); t.peer_map = dv.alloc<u32>(NP);
    t.dcont = dv.alloc<DocContainer>(NC + 1, true); t.cid_map = dv.alloc<u32>(NC);
    t.dkey_off = dv.alloc<u64>(NK); t.dkey_len = dv.alloc<u32>(NK); t.key_map = dv.alloc<u32>(NK);
    t.blk_order = dv.alloc<u32>(n.blocks);
    t.ch_order = dv.alloc<u32>(NCH); t.ch_aorder = dv.alloc<u32>(NCH); t.ch_peer = dv.alloc<u16>(NCH);
    t.ch_applied = dv.alloc<u8>(NCH, true); t.ch_lamport = dv.alloc<u32>(NCH, true); t.ch_walk = dv.alloc<u32>(NCH);
    t.ch_pos = dv.alloc<u32>(NCH, true); t.ch_trim = dv.alloc<u32>(NCH, true);
    // status of multi-blob documents (import_batch groups, lb_docset_import): per-copy epochs, per-blob pending hulls
    i32* d_pend_scratch = nullptr;
    if (b->n_blobs > D) {
        t.ch_epoch = dv.alloc<u32>(NCH);
        t.ch_maxend = dv.alloc<i32>(NCH);
        t.head_lamport = dv.alloc<u32>(NP);
        d_pend_scratch = dv.alloc<i32>(2 * (u64)b->n_blobs + 2);
    }
    LB_BATCH_LAUNCH(b, k_doc_tables, nblk(D, 64), 64, 0, t.bytes, b->d_docs, D, t.blocks, t);
    u32* d_vv_cells = dv.alloc<u32>(D + 1);
    LB_BATCH_LAUNCH(b, k_doc_vv_cells, nblk(D), TPB, 0, b->d_docs, D, d_vv_cells);
    run_scans(b, {scan_job(d_vv_cells, b->d_docs, &DocInfo::vv0, D)});
    u64 VV = d2h_one(b, &b->d_docs[D].vv0);
    t.ch_vv = dv.alloc<i32>(VV);
    u32* d_cursor = dv.alloc<u32>(NP);
    LB_BATCH_LAUNCH(b, k_doc_causal, nblk(D, 64), 64, 0, b->d_docs, D, t.blocks, t, d_cursor, ln.doc_blob0, d_pend_scratch);
    LB_BATCH_LAUNCH(b, k_doc_frontiers, nblk(D, 64), 64, 0, b->d_docs, D, t);
    if (ln.ck_range) {
        t.ck_end = dv.alloc<i32>(NP + 1);
        LB_BATCH_LAUNCH(b, k_doc_checkout, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, t, ln.ck_range, ln.ck_peer, ln.ck_ctr);
    }
    u32* d_atoms = dv.alloc<u32>(D + 1);
    u32* d_mapslots = dv.alloc<u32>(D + 1);
    LB_BATCH_LAUNCH(b, k_doc_atoms_mapslots, nblk(D), TPB, 0, b->d_docs, D, d_atoms, d_mapslots);
    run_scans(b, {scan_job(d_atoms, b->d_docs, &DocInfo::atom0, D), scan_job(d_mapslots, b->d_docs, &DocInfo::mapslot0, D)});
    DocInfo dtot = d2h_one(b, &b->d_docs[D]);
    n.atoms = dtot.atom0;
    n.map_slots = dtot.mapslot0;
    mark(b, EV_RESOLVE);
}

// phase 4: classify + map LWW, then the capacities of the sequence trackers' pools
void phase_classify(lb_batch* b) {
    Dev& dv = b->dev; BatchTables& t = b->tb; BatchSizes& n = b->n; const u32 D = (u32)b->n_docs;
    const u64 NR = n.rows, NTR = n.tree_ops, NC = n.cids;
    t.tr_rec = dv.alloc<uint4>(NTR); t.tr_key = dv.alloc<u64>(NTR); t.tr_ids = dv.alloc<uint4>(NTR);
    t.op_kind = dv.alloc<u8>(NR); t.op_cidx = dv.alloc<u32>(NR); t.op_lamport = dv.alloc<u32>(NR);
    t.atom_row = dv.alloc<u32>(n.atoms);
    t.op_rec = dv.alloc<uint4>(NR); t.op_aux = dv.alloc<u32>(NR);
    t.map_best = dv.alloc<unsigned long long>(n.map_slots, true);
    t.map_row = dv.alloc<u32>(n.map_slots);
    if (NR) {
        LB_BATCH_LAUNCH(b, k_op_classify, nblk(NR, 256), 256, 0, b->d_docs, NR, t);
        LB_BATCH_LAUNCH(b, k_map_winner, nblk(NR, 256), 256, 0, b->d_docs, NR, t);
    }
    // capacities -> pools
    u32* cap_leaf = dv.alloc<u32>(NC + 1, true); u32* cap_node = dv.alloc<u32>(NC + 1, true);
    u32* cap_out = dv.alloc<u32>(NC + 1, true); u32* cap_cvv = dv.alloc<u32>(NC + 1, true);
    u32* span_cap = dv.alloc<u32>(D + 1, true);
    LB_BATCH_LAUNCH(b, k_container_caps, nblk(D), TPB, 0, b->d_docs, D, t.dcont, cap_leaf, cap_node, cap_out, cap_cvv, span_cap, SEQ_LEAF_W);
    run_scans(b, {scan_job(cap_leaf, t.dcont, &DocContainer::leaf0, NC), scan_job(cap_node, t.dcont, &DocContainer::node0, NC),
                  scan_job(cap_out, t.dcont, &DocContainer::out0, NC), scan_job(cap_cvv, t.dcont, &DocContainer::cvv0, NC),
                  scan_job(span_cap, b->d_docs, &DocInfo::span0, D)});
    DocContainer ctot = d2h_one(b, t.dcont + NC);
    n.leaves = ctot.leaf0; n.nodes = ctot.node0; n.runs = ctot.out0; n.cvv = ctot.cvv0;
    mark(b, EV_CLASSIFY);
}

// phase 5: sequence integration; with LB_FLAG_CURSORS the ropes' order is kept for lb_batch_cursor_pos (k_cursor.cuh)
void phase_integrate(lb_batch* b) {
    Dev& dv = b->dev; cudaStream_t st = dv.stream; BatchTables& t = b->tb; const BatchSizes& n = b->n; const u32 D = (u32)b->n_docs;
    const u64 NATOM = n.atoms, NOUT = n.runs, NC = n.cids;
    SeqPools sp;
    memset(&sp, 0, sizeof(sp));
    sp.leaf = dv.alloc<uint4>(n.leaves * SEQ_LEAF_W); sp.node = dv.alloc<uint2>(n.nodes * SEQ_LEAF_W);
    sp.node_parent = dv.alloc<u32>(n.nodes); sp.atom_leaf = dv.alloc<u32>(NATOM);
    CK(cudaMemsetAsync(sp.atom_leaf, 0xFF, sizeof(u32) * NATOM, st));   // LEAF_NONE everywhere
    sp.a_org = dv.alloc<uint4>(NATOM); sp.cvv = dv.alloc<i32>(n.cvv, true);
    sp.cont_epoch = dv.alloc<u32>(NC + 1); sp.next_doc = dv.alloc<u32>(1, true);
    t.out_row = dv.alloc<u32>(NOUT); t.out_off = dv.alloc<u32>(NOUT); t.out_len = dv.alloc<u32>(NOUT);
    const unsigned seq_ctas = seq_resident_ctas(b->dev.device);
    if (nblk(D, LB_SEQ_WARPS) > seq_ctas) LB_BATCH_LAUNCH(b, k_seq_integrate<1>, seq_ctas, 32 * LB_SEQ_WARPS, 0, b->d_docs, D, sp, t);
    else LB_BATCH_LAUNCH(b, k_seq_integrate<0>, nblk(D, LB_SEQ_WARPS), 32 * LB_SEQ_WARPS, 0, b->d_docs, D, sp, t);
    mark(b, EV_INTEGRATE);
    if (b->flags & LB_FLAG_CURSORS) {
        if (NOUT >= 0xFFFFFFFFull) { g_last_error = "batch too large for LB_FLAG_CURSORS: spans must fit 32 bits"; throw lb_status(LB_ERR_INVALID_ARG); }
        b->cur.ord = dv.alloc<uint4>(NOUT);
        b->cur.idx = dv.alloc<uint2>(NOUT);
        b->cur.n = dv.alloc<u32>(NC + 1, true);
        u32* ent_cont = dv.alloc<u32>(NOUT);
        u32* fill = dv.alloc<u32>(NC + 1, true);
        // the atom -> leaf array is done with: it holds the span marks of the counting sort now
        CK(cudaMemsetAsync(sp.atom_leaf, 0xFF, sizeof(u32) * NATOM, st));
        LB_BATCH_LAUNCH(b, k_cursor_tables, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, sp, t, b->cur, sp.atom_leaf,
                        ent_cont, fill);
        dv.release(ent_cont); dv.release(fill);
    }
    if (!(b->flags & LB_FLAG_KEEP_DEVICE)) {   // the tracker pools are the largest tables of the batch: free them early
        dv.release(sp.leaf); dv.release(sp.node); dv.release(sp.node_parent); dv.release(sp.atom_leaf); dv.release(sp.a_org);
        dv.release(sp.cvv); dv.release(sp.cont_epoch); dv.release(sp.next_doc); dv.release(t.atom_row); dv.release(t.op_rec);
    }
    mark(b, EV_CURSORS);
}

// phase 5b: movable trees
void phase_tree(lb_batch* b) {
    Dev& dv = b->dev; BatchTables& t = b->tb; const u32 D = (u32)b->n_docs;
    const u64 NTR = b->n.tree_ops;
    if (NTR) {
        u32* d_tree_slots = dv.alloc<u32>(D + 1);
        u32* d_max_tree_atoms = dv.alloc<u32>(1, true);
        LB_BATCH_LAUNCH(b, k_doc_tree_slots, nblk(D), TPB, 0, b->d_docs, D, d_tree_slots, d_max_tree_atoms);
        run_scans(b, {scan_job(d_tree_slots, b->d_docs, &DocInfo::tree0, D)});
        u64 NTS = d2h_one(b, &b->d_docs[D].tree0);
        const u32 max_atoms = d2h_one(b, d_max_tree_atoms);
        t.ts_key = dv.alloc<u64>(NTR); t.ts_val = dv.alloc<u32>(NTR); t.ts_rec = dv.alloc<uint4>(NTR);
        t.tn_parent = dv.alloc<u32>(NTS); t.tn_move = dv.alloc<u32>(NTS); t.tn_base = dv.alloc<u32>(NTS);
        t.tn_cnt = dv.alloc<u32>(NTS); t.tn_sib = dv.alloc<u32>(NTS); t.ns_key = dv.alloc<u64>(NTS); t.tn_child = dv.alloc<u32>(NTS);
        t.tn_root = dv.alloc<u32>(NTS); t.tn_aopen = dv.alloc<u32>(NTS); t.tn_aclose = dv.alloc<u32>(NTS);
        // 16-bit parent links of one document in shared memory, sized for the largest tree document of the batch:
        // the number of resident documents (one sequential chain each) is what the apply kernel's speed depends on
        u32 s_nodes = max_atoms < TREE_S_NODES_MAX ? max_atoms : (u32)TREE_S_NODES_MAX;
        s_nodes = (s_nodes + 63u) & ~63u;
        const size_t tree_smem = (size_t)TREE_WARPS * s_nodes * sizeof(u16);
#ifndef LB_SIMT_EMU
        CK(cudaFuncSetAttribute(k_tree_apply, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tree_smem));
        CK(cudaFuncSetAttribute(k_tree_apply, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        if (phase_trace()) {
            int nb = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_tree_apply, 32 * TREE_WARPS, tree_smem);
            fprintf(stderr, "[trace] k_tree_apply: %zu bytes of shared memory per document, %d documents resident per SM\n", tree_smem, nb);
        }
#endif
        LB_BATCH_LAUNCH(b, k_tree_sort, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, t);
        LB_BATCH_LAUNCH(b, k_tree_apply, nblk((u64)D * 32, 32 * TREE_WARPS), 32 * TREE_WARPS, tree_smem, b->d_docs, D, t, s_nodes);
        LB_BATCH_LAUNCH(b, k_tree_layout, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, t);
    }
    mark(b, EV_TREE);
    b->timings.tree_ops = NTR;
}

// phase 6: every document's JSON and state hash.  The host-buffer entry point sends the JSON home from here, on a
// second stream, while the later phases compute.
void phase_materialise(lb_batch* b, PhaseLinks& ln) {
    Dev& dv = b->dev; BatchTables& t = b->tb; const u32 D = (u32)b->n_docs;
    ln.acc = dv.alloc<unsigned long long>(4, true);
    if (!(b->flags & LB_FLAG_NO_JSON)) {
        LB_BATCH_LAUNCH(b, k_json, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, t, (u8*)nullptr, 0);
        u32* d_json_padded = dv.alloc<u32>(D + 1);
        LB_BATCH_LAUNCH(b, k_json_padlen, nblk(D), TPB, 0, b->d_docs, D, d_json_padded);
        run_scans(b, {scan_job(d_json_padded, b->d_docs, &DocInfo::json_off, D)});
        b->json.total = d2h_one(b, &b->d_docs[D].json_off);
        b->json.d = dv.alloc<u8>(b->json.total + 16, true);
        LB_BATCH_LAUNCH(b, k_json, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, t, b->json.d, 1);
    }
    LB_BATCH_LAUNCH(b, k_doc_hash, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, (const u8*)b->json.d, ln.acc);
    mark(b, EV_MATERIALISE);
    if (b->eager_json && b->json.total && !(b->flags & LB_FLAG_NO_JSON)) {
        CK(cudaStreamCreate(&b->stream2));
        CK(cudaEventCreate(&b->json_ev));
        CK(cudaEventRecord(b->json_ev, dv.stream));
        b->json.host = (char*)lbstage::host_cache().take(b->json.total + 1);   // taken here: no memory fails the import
        if (!b->json.host) { g_last_error = "out of host memory"; throw lb_status(LB_ERR_OOM); }
        b->json_thread = std::thread([b] {
            b->json_ok = cudaSetDevice(b->dev.device) == cudaSuccess && cudaStreamWaitEvent(b->stream2, b->json_ev, 0) == cudaSuccess &&
                         b->json.fetch(b->stream2, "json d2h failed") == LB_OK;
        });
    }
}

// phase 6b: attribution (reads out_*, map_*, tn_*)
void phase_attribution(lb_batch* b) {
    if (b->flags & LB_FLAG_ATTRIBUTION) {
        Dev& dv = b->dev; const u32 D = (u32)b->n_docs;
        u32* cord = dv.alloc<u32>(b->n.cids + 1);
        u32* kord = dv.alloc<u32>(b->n.keys + 1);
        u32* d_attr_len = dv.alloc<u32>(D + 1);
        b->d_attr_off = dv.alloc<u64>(D + 1);
        LB_BATCH_LAUNCH(b, k_attr, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, b->tb, cord, kord, d_attr_len,
                        (const u64*)nullptr, (u8*)nullptr, 0);
        run_scans(b, {scan_job(d_attr_len, b->d_attr_off, D)});
        b->attr.total = d2h_one(b, b->d_attr_off + D);
        b->attr.d = dv.alloc<u8>(b->attr.total + 16);
        LB_BATCH_LAUNCH(b, k_attr, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, b->tb, cord, kord, d_attr_len,
                        (const u64*)b->d_attr_off, b->attr.d, 1);
    }
    mark(b, EV_ATTRIBUTION);
}

// phase 7: re-export (all_updates per document)
void phase_export(lb_batch* b) {
    if (b->flags & LB_FLAG_EXPORT) {
        Dev& dv = b->dev; cudaStream_t st = dv.stream; BatchTables& t = b->tb; const u32 D = (u32)b->n_docs;
        const u64 NCH = b->n.changes, NR = b->n.rows, NTR = b->n.tree_ops, NPOS = b->n.pos;
        trace_point(b, "before export");
        if (NTR) {
            t.pos_rank = dv.alloc<u32>(NPOS); t.pos_rep = dv.alloc<u32>(NPOS);
            t.ps_key = dv.alloc<u64>(NPOS); t.ps_val = dv.alloc<u32>(NPOS);
        }
        t.x_rec = dv.alloc<uint4>(NR); t.r_bytes = dv.alloc<u32>(NR); t.r_flag = dv.alloc<u8>(NR);
        t.ch_nseg = dv.alloc<u32>(NCH + 1, true); t.ch_novf = dv.alloc<u32>(NCH + 1, true);
        t.ch_seg0 = dv.alloc<u64>(NCH + 2, true);
        t.n_changes = NCH; t.n_rows = NR;
        t.ch_syn = dv.alloc<u32>(NCH + 1, true); t.ch_syn0 = dv.alloc<u64>(NCH + 2, true);
        t.xdoc = dv.alloc<XDoc>(D + 1, true);
        t.ch_aval = dv.alloc<u32>(NCH + 1, true); t.ch_astr = dv.alloc<u32>(NCH + 1, true);
        t.ch_aval0 = dv.alloc<u64>(NCH + 2, true); t.ch_astr0 = dv.alloc<u64>(NCH + 2, true);
        // segment / final-change records: one slot per change + one per extra segment of a split change; the
        // extras are counted by k_exp_changes, so the arrays are sized with a bound first and checked after the scan
        u64 SEGCAP = NCH + NCH / 4 + 1024;
        if (getenv("LB_EXPORT_TIGHT_SEGCAP")) SEGCAP = NCH;   // testing hook: force the growth path
        // the u32 tables of the two groups (SG_TABLES, FC_TABLES) in allocation order; the *_skip and fc_tail tables
        // start zeroed, and fc_block (the one byte-wide table) has its place before fc_skip
        for (auto m : SG_TABLES) t.*m = dv.alloc<u32>(SEGCAP, m == &BatchTables::sg_skip);
        for (auto m : FC_TABLES) {
            if (m == &BatchTables::fc_skip) t.fc_block = dv.alloc<u8>(SEGCAP);
            t.*m = dv.alloc<u32>(SEGCAP, m == &BatchTables::fc_skip || m == &BatchTables::fc_tail);
        }
        b->fc_cap = SEGCAP;
        trace_point(b, "export allocs");
        LB_BATCH_LAUNCH(b, k_exp_init, nblk(D), TPB, 0, b->d_docs, D, t);
        if (NTR) LB_BATCH_LAUNCH(b, k_exp_posrank, nblk((u64)D * 32, 128), 128, 0, b->d_docs, D, t);
        if (NCH) LB_BATCH_LAUNCH(b, k_exp_arena, nblk(NCH * 32, XCH_TPB), XCH_TPB, 0, NCH, t, b->d_docs);
        run_scans(b, {scan_job(t.ch_aval, t.ch_aval0, NCH), scan_job(t.ch_astr, t.ch_astr0, NCH)});
        trace_point(b, "posrank+arena");
        if (NCH) LB_BATCH_LAUNCH(b, k_exp_changes, nblk(NCH * 32, XCH_TPB), XCH_TPB, 0, b->d_docs, NCH, t);
        trace_point(b, "changes pass 0");
        run_scans(b, {scan_job(t.ch_novf, t.ch_seg0, NCH), scan_job(t.ch_syn, t.ch_syn0, NCH)});
        u64 NOVF = d2h_one(b, t.ch_seg0 + NCH);
        u64 NSYN = d2h_one(b, t.ch_syn0 + NCH);
        t.has_syn = NSYN ? 1 : 0;
        t.s_rec = dv.alloc<uint4>(NSYN); t.s_len = dv.alloc<u32>(NSYN); t.s_bytes = dv.alloc<u32>(NSYN);
        t.s_flag = dv.alloc<u8>(NSYN); t.s_voff = dv.alloc<u64>(NSYN); t.s_vlen = dv.alloc<u32>(NSYN); t.s_aux = dv.alloc<u32>(NSYN);
        if (NCH + NOVF > SEGCAP) {   // unusually many split changes: grow the tables, keep what k_exp_changes wrote
            for (auto m : SG_TABLES) {
                u32* nw = dv.alloc<u32>(NCH + NOVF);
                CK(cudaMemcpyAsync(nw, t.*m, sizeof(u32) * NCH, cudaMemcpyDeviceToDevice, st));
                dv.release(t.*m);
                t.*m = nw;
            }
        }
        grow_fc_tables(b, NCH + NOVF);
        b->n_segs = NCH + NOVF;
        if (NOVF) LB_BATCH_LAUNCH(b, k_exp_split_changes, nblk(NCH, 64), 64, 0, b->d_docs, NCH, t);
        LB_BATCH_LAUNCH(b, k_exp_store, nblk(D, 64), 64, 0, b->d_docs, D, t);
        b->exported.d = export_encode(b, t, &b->exported.total, false);
        b->timings.export_bytes = b->exported.total;
    }
    mark(b, EV_EXPORT);
}

// the documents' records, the counters and the documents' peer entries to the host
void results_to_host(lb_batch* b, const PhaseLinks& ln) {
    Dev& dv = b->dev; cudaStream_t st = dv.stream; const BatchTables& t = b->tb; const u32 D = (u32)b->n_docs;
    b->t_tail = std::chrono::steady_clock::now();
    b->docs.resize(D + 1);
    CK(cudaMemcpyAsync(b->docs.data(), b->d_docs, sizeof(DocInfo) * (D + 1), cudaMemcpyDeviceToHost, st));
    unsigned long long acc[4];
    CK(cudaMemcpyAsync(acc, ln.acc, sizeof(acc), cudaMemcpyDeviceToHost, st));
    unsigned long long dws[4] = {0, 0, 0, 0};
    CK(cudaMemcpyAsync(dws, t.dw_stats, sizeof(dws), cudaMemcpyDeviceToHost, st));
    if (t.xdoc) {
        b->xdocs.resize(D);
        CK(cudaMemcpyAsync(b->xdocs.data(), t.xdoc, sizeof(XDoc) * D, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    // the peer table is sized by the blocks' peer registers (a few entries per BLOCK: hundreds of MB for 10^6 blocks) but a
    // document uses only its first P entries: those are packed on the device and only they travel
    b->peer_base.assign(D + 1, 0);
    for (u32 d = 0; d < D; d++) b->peer_base[d + 1] = b->peer_base[d] + b->docs[d].P;
    const u64 total = b->peer_base[D];
    b->dpeer.resize(total);
    if (total) {
        u64* d_pbase = dv.alloc<u64>(D + 1);
        DocPeer* d_packed = dv.alloc<DocPeer>(total);
        CK(cudaMemcpyAsync(d_pbase, b->peer_base.data(), sizeof(u64) * (D + 1), cudaMemcpyHostToDevice, st));
        LB_BATCH_LAUNCH(b, k_pack_peers, nblk(D), TPB, 0, b->d_docs, D, t.dpeer, d_pbase, d_packed);
        CK(cudaMemcpyAsync(b->dpeer.data(), d_packed, sizeof(DocPeer) * total, cudaMemcpyDeviceToHost, st));
    }
    mark(b, EV_D2H);   // the result copies are queued
    CK(cudaStreamSynchronize(st));
    lb_counters& c = b->counters;
    c.docs = D; c.docs_ok = acc[3]; c.atom_ops = acc[1]; c.pending_changes = acc[2]; c.state_hash = acc[0];
    c.blocks = b->n.blocks; c.changes = b->n.changes; c.op_rows = b->n.rows;
    lb_timings& tm = b->timings;
    tm.decode_fast_blocks = dws[0]; tm.decode_lane_blocks = dws[1]; tm.decode_unstaged_blocks = dws[2];
    c.json_bytes = 0;
    for (u32 d = 0; d < D; d++) c.json_bytes += b->docs[d].json_len;
}

void pipeline(lb_batch* b) {
    if (b->n_docs == 0) {
        b->docs.resize(1);
        return;
    }
    PhaseLinks ln;
    phase_frame(b, ln);
    phase_decode(b);
    phase_resolve(b, ln);
    phase_classify(b);
    phase_integrate(b);
    phase_tree(b);
    phase_materialise(b, ln);
    phase_attribution(b);
    phase_export(b);
    results_to_host(b, ln);
}

// ImportStatus / vv / frontiers spans of every document, flat: [off[d], off[d + 1]) of one array per kind (a vector per
// document and kind cost ~0.1 s of host time per 10^5-document batch in allocations alone)
void build_status(lb_batch* b) {
    size_t D = b->n_docs;
    for (int k = 0; k < 4; k++) { b->span_off[k].assign(D + 1, 0); b->spans[k].clear(); }
    size_t total_peers = 0;
    for (size_t d = 0; d < D; d++) total_peers += b->docs[d].P;
    for (int k = 0; k < 4; k++) b->spans[k].reserve(k == 1 ? 16 : total_peers);
    for (size_t d = 0; d < D; d++) {
        DocInfo& di = b->docs[d];
        if (di.code == DOC_OK && di.has_unsupported) di.code = DOC_ERR_UNSUPPORTED;
        if (di.code == DOC_OK || di.code == DOC_ERR_UNSUPPORTED || di.code == DOC_ERR_FRONTIERS) {
            for (u32 p = 0; p < di.P; p++) {
                const DocPeer& dp = b->dpeer[b->peer_base[d] + p];
                if (dp.has_succ && !b->stored_only) b->spans[0].push_back(lb_id_span{dp.id, dp.succ_lo, dp.end_counter});
                if (dp.pend_hi > dp.pend_lo && !b->stored_only) b->spans[1].push_back(lb_id_span{dp.id, dp.pend_lo, dp.pend_hi});
                if (dp.end_counter > 0) b->spans[2].push_back(lb_id_span{dp.id, 0, dp.end_counter});
                if (dp.is_head && dp.end_counter > 0) b->spans[3].push_back(lb_id_span{dp.id, dp.end_counter - 1, dp.end_counter});
            }
        }
        for (int k = 0; k < 4; k++) b->span_off[k][d + 1] = b->spans[k].size();
    }
}

void timings_from_events(lb_batch* b) {
    auto el = [&](BatchEvent a, BatchEvent c) {   // 0 when either end was not recorded (the empty batch)
        float ms = 0;
        if (b->ev_recorded[a] && b->ev_recorded[c]) cudaEventElapsedTime(&ms, b->ev[a], b->ev[c]);
        return ms;
    };
    lb_timings& t = b->timings;
    t.h2d = el(EV_START, EV_H2D);
    t.frame = el(EV_H2D, EV_FRAME);
    t.decode = el(EV_FRAME, EV_DECODE);
    t.resolve = el(EV_DECODE, EV_RESOLVE);
    t.classify = el(EV_RESOLVE, EV_CLASSIFY);
    t.integrate = el(EV_CLASSIFY, EV_INTEGRATE);
    t.cursors = el(EV_INTEGRATE, EV_CURSORS);
    t.tree = el(EV_CURSORS, EV_TREE);
    t.materialise = el(EV_TREE, EV_MATERIALISE);
    t.attribution = el(EV_MATERIALISE, EV_ATTRIBUTION);
    t.reexport = el(EV_ATTRIBUTION, EV_EXPORT);
    t.d2h = el(EV_EXPORT, EV_D2H);
    t.total_device = el(EV_H2D, EV_EXPORT);
}

lb_status run_batch(lb_batch* b) {
    try {
        pipeline(b);
        build_status(b);
        timings_from_events(b);
        auto now = std::chrono::steady_clock::now();
        b->timings.host_call_ms = std::chrono::duration<float, std::milli>(now - b->t_call).count();
        b->timings.host_tail_ms = std::chrono::duration<float, std::milli>(now - b->t_tail).count();
    } catch (lb_status s) {
        return s;
    }
    return LB_OK;
}

// host-side peek at a blob (only what import_batch's ordering needs: mode and the number of changes)
u32 blob_mode(const uint8_t* p, size_t n) { return n >= 22 ? ((u32)p[20] << 8) | p[21] : 0xFFFFu; }
u64 blob_change_count(const uint8_t* p, size_t n) {
    if (n < 22) return 0;
    size_t i = 22;
    auto varint = [&](u64* v) {
        *v = 0;
        for (int s = 0; s < 70 && i < n; s += 7) {
            uint8_t c = p[i++];
            *v |= (u64)(c & 0x7f) << (s < 64 ? s : 63);
            if (!(c & 0x80)) return true;
        }
        return false;
    };
    u64 total = 0;
    while (i < n) {
        u64 len, x;
        if (!varint(&len) || len > n - i) break;
        size_t end = i + (size_t)len;
        bool ok = true;
        for (int k = 0; k < 5 && ok; k++) ok = varint(&x) && i <= end;
        if (ok) total += x;   // the fifth varint of the envelope is n_changes
        i = end;
    }
    return total;
}

lb_status check_device(const lb_options* opt) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
        g_last_error = "no CUDA device: loro_b200 has no CPU fallback";
        return LB_ERR_NO_DEVICE;
    }
    int dev = opt ? opt->device : 0;
    if (dev < 0 || dev >= n) {
        g_last_error = "bad device ordinal";
        return LB_ERR_INVALID_ARG;
    }
    if (cudaSetDevice(dev) != cudaSuccess) {
        g_last_error = "cudaSetDevice failed";
        return LB_ERR_CUDA;
    }
#ifndef LB_SIMT_EMU
    {   // keep freed table memory cached in the stream-ordered pool between batches
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            unsigned long long thr = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
    }
#endif
    return LB_OK;
}

// What every import entry point does around its own part: the device check, a batch with its stream and events, then
// `fill` (it builds the blob list, ends in upload_and_run and returns a status or throws one), and the one place where a
// failed batch is freed and a good one handed out.
template <class Fill>
lb_status import_with_new_batch(const lb_options* opt, lb_batch** out, Fill fill) {
    lb_status s = check_device(opt);
    if (s != LB_OK) return s;
    lb_batch* b = new lb_batch();
    b->flags = opt ? opt->flags : 0;
    b->dev.device = opt ? opt->device : 0;
    try {
        b->dev.stream = stream_take(b->dev.device);
        if (!b->dev.stream) { g_last_error = "cudaStreamCreate failed"; throw lb_status(LB_ERR_CUDA); }
        for (cudaEvent_t& e : b->ev) CK(cudaEventCreate(&e));
        b->ev_created = true;
        s = fill(b);
    } catch (lb_status e) {
        s = e;
    }
    if (s != LB_OK) { lb_batch_free(b); return s; }
    *out = b;
    return LB_OK;
}

// The blob table (offsets and lengths into `d_bytes`, already on the device) goes up, then the pipeline runs.
lb_status upload_and_run(lb_batch* b, const std::vector<u64>& offs, const std::vector<u32>& lens, const u8* d_bytes) {
    const size_t Q = b->n_blobs;
    b->d_offs = b->dev.alloc<u64>(Q + 1);
    b->d_lens = b->dev.alloc<u32>(Q + 1);
    CK(cudaMemcpyAsync(b->d_offs, offs.data(), sizeof(u64) * (Q + 1), cudaMemcpyHostToDevice, b->dev.stream));
    CK(cudaMemcpyAsync(b->d_lens, lens.data(), sizeof(u32) * (Q + 1), cudaMemcpyHostToDevice, b->dev.stream));
    b->tb.bytes = d_bytes;
    b->timings.decode_bytes_read = b->counters.blob_bytes;
    mark(b, EV_H2D);
    return run_batch(b);
}

const char* const ERR_FAILED_DOC = "document failed to import";
const char* const ERR_NOT_COVERED = "document uses features the export phase does not cover";
// the answer for a document whose code is not OK: one with ops the engine does not merge (LB_DOC_ERR_UNSUPPORTED) is not
// covered by the export phase either; any other code means the import failed
lb_exports::Answer doc_error(const DocInfo& di) {
    if (di.code == DOC_ERR_UNSUPPORTED) return lb_exports::Answer{LB_ERR_UNSUPPORTED, ERR_NOT_COVERED, nullptr, 0};
    return lb_exports::Answer{LB_ERR_INVALID_ARG, ERR_FAILED_DOC, nullptr, 0};
}

// The start of an on-demand export pass over the documents h_req marks: a copy of the batch's tables with the request
// mask (x_req) and a fresh XDoc table, and the marked documents' changes prepared for the stores (k_exp_init,
// k_exp_changes, k_exp_split_changes).  The caller releases xt.x_req and xt.xdoc.
BatchTables export_pass(lb_batch* b, const std::vector<u8>& h_req) {
    Dev& dv = b->dev;
    const u32 D = (u32)b->n_docs;
    const u64 NCH = b->n.changes;
    BatchTables xt = b->tb;
    u8* d_req = dv.alloc<u8>(D);
    CK(cudaMemcpyAsync(d_req, h_req.data(), D, cudaMemcpyHostToDevice, dv.stream));
    xt.x_req = d_req;
    xt.xdoc = dv.alloc<XDoc>(D + 1, true);
    LB_BATCH_LAUNCH(b, k_exp_init, nblk(D), TPB, 0, b->d_docs, D, xt);
    if (NCH) {
        LB_BATCH_LAUNCH(b, k_exp_changes, nblk(NCH * 32, XCH_TPB), XCH_TPB, 0, b->d_docs, NCH, xt);
        LB_BATCH_LAUNCH(b, k_exp_split_changes, nblk(NCH, 64), 64, 0, b->d_docs, NCH, xt);
    }
    return xt;
}

// One pass of the export of chosen id spans (change_store.rs:179-199 export_blocks_in_range, :494-528
// export_blocks_from) over the documents of a round, one span set each: the import store of each marked document is
// rebuilt, its changes are cut to the document's spans (Change::slice at both ends) on their way into a fresh export
// store, and the result is encoded like the import-time export.  The phase-7 tables of the batch are reused; only the
// per-pass pieces (span table, request mask, block list, scratch, output) are allocated.  The stores rewrite the rows'
// flags (k_exp_store merges ops across changes), which is why a document can be in one request per pass only.
// h_span0 / h_spans: the span table over the batch's peer slots (BatchTables::x_span0); cuts: some span ends below its
// peer's vv; h_req: the request mask.
// Returns the round's packed blobs in host memory, with the XDoc table that places them (exp_off / exp_len of every
// marked document).
std::unique_ptr<uint8_t[]> export_round(lb_batch* b, const std::vector<u32>& h_span0, const std::vector<XSpan>& h_spans,
                                        bool cuts, const std::vector<u8>& h_req, std::vector<XDoc>& xd) {
    Dev& dv = b->dev;
    cudaStream_t st = dv.stream;
    const u32 D = (u32)b->n_docs;
    grow_fc_tables(b, b->n_segs + h_spans.size());   // a document's final changes get one slot per segment and one per span (xfc0)
    u32* d_span0 = dv.alloc<u32>(h_span0.size());
    XSpan* d_spans = dv.alloc<XSpan>(std::max<size_t>(h_spans.size(), 1));
    CK(cudaMemcpyAsync(d_span0, h_span0.data(), sizeof(u32) * h_span0.size(), cudaMemcpyHostToDevice, st));
    if (!h_spans.empty()) CK(cudaMemcpyAsync(d_spans, h_spans.data(), sizeof(XSpan) * h_spans.size(), cudaMemcpyHostToDevice, st));
    BatchTables xt = export_pass(b, h_req);
    CK(cudaStreamSynchronize(st));   // pageable host memory
    xt.x_span0 = d_span0;
    xt.x_spans = d_spans;
    LB_BATCH_LAUNCH(b, k_exp_store, nblk(D, 64), 64, 0, b->d_docs, D, xt);
    u64 XT = 0;
    u8* d_out = export_encode(b, xt, &XT, cuts);
    xd.resize(D);
    CK(cudaMemcpyAsync(xd.data(), xt.xdoc, sizeof(XDoc) * D, cudaMemcpyDeviceToHost, st));
    std::unique_ptr<uint8_t[]> out(new uint8_t[XT + 1]);
    if (!lbstage::download(d_out, out.get(), XT, st)) { g_last_error = "export d2h failed"; throw lb_status(LB_ERR_CUDA); }
    CK(cudaStreamSynchronize(st));
    dv.release(d_span0); dv.release(d_spans); dv.release(xt.x_req); dv.release(xt.xdoc); dv.release(d_out);
    return out;
}

// A document's span set in the form export_span_sets compares and lays out: per peer slot p of the document, the number
// of its spans, then (start, end, fresh) of each, sorted by start.
using SpanKey = std::vector<i32>;
const char* const ERR_SPANS_OVERLAP = "two spans of one peer overlap (the reference would store their changes twice or panic)";
const char* const ERR_SPANS_GAP = "a span starts above an earlier-listed span of its peer that does not end at its start "
                                  "(the reference panics: counter should be continuous)";

// Answers requests that each name a document and a span set.  key_of(i, di, peers, key) writes request i's key and
// returns nullptr, or returns why the request is refused.  Equal keys of one document are answered once, the key that
// selects [0, vv) of every peer from the import-time export (no launch), and the rest in rounds: round r holds the r-th
// distinct key of every document, so the number of passes is the largest number of distinct span sets asked of one
// document, whatever the number of documents or spans.
template <class DocOf, class KeyOf>
void export_span_sets(lb_batch* b, size_t n, DocOf doc_of, KeyOf key_of, lb_exports& e) {
    struct Version { size_t doc; u32 round; SpanKey key; };
    std::vector<Version> versions;                          // distinct (document, key) pairs, round by round below
    std::unordered_map<size_t, std::vector<u32>> of_doc;    // document -> its versions, in order of first request
    std::vector<u32> version_of(n, ~0u);                    // request -> version; ~0: all_updates or an error
    e.answers.assign(n, lb_exports::Answer{LB_OK, nullptr, nullptr, 0});
    std::vector<size_t> all_updates;                        // requests answered by the import-time export
    for (size_t i = 0; i < n; i++) {
        const size_t doc = doc_of(i);
        const DocInfo& di = b->docs[doc];
        if (di.code != DOC_OK) { e.answers[i] = doc_error(di); continue; }
        const DocPeer* dp = &b->dpeer[b->peer_base[doc]];
        SpanKey key, whole;
        if (const char* err = key_of(i, di, dp, key)) { e.answers[i] = lb_exports::Answer{LB_ERR_INVALID_ARG, err, nullptr, 0}; continue; }
        for (u32 p = 0; p < di.P; p++) {
            if (dp[p].end_counter > 0) whole.insert(whole.end(), {1, 0, dp[p].end_counter, 1});
            else whole.push_back(0);
        }
        if (key == whole) { all_updates.push_back(i); continue; }
        std::vector<u32>& mine = of_doc[doc];
        for (u32 v : mine) if (versions[v].key == key) version_of[i] = v;
        if (version_of[i] == ~0u) {
            version_of[i] = (u32)versions.size();
            versions.push_back(Version{doc, (u32)mine.size(), std::move(key)});
            mine.push_back(version_of[i]);
        }
    }
    // all_updates: the document's blob of the import-time export, copied out of the batch's export buffer
    if (!all_updates.empty()) {
        u64 total = 0;
        for (size_t i : all_updates) total += b->xdocs[doc_of(i)].exp_len;
        e.bufs.emplace_back(new uint8_t[total + 1]);
        uint8_t* w = e.bufs.back().get();
        for (size_t i : all_updates) {
            const XDoc& x = b->xdocs[doc_of(i)];
            if ((x.flags & 1) || x.exp_len == 0) { e.answers[i] = lb_exports::Answer{LB_ERR_UNSUPPORTED, ERR_NOT_COVERED, nullptr, 0}; continue; }
            CK(cudaMemcpyAsync(w, b->exported.d + x.exp_off, x.exp_len, cudaMemcpyDeviceToHost, b->dev.stream));
            e.answers[i].bytes = w;
            e.answers[i].len = x.exp_len;
            w += x.exp_len;
        }
        CK(cudaStreamSynchronize(b->dev.stream));
    }
    size_t rounds = 0;
    for (const auto& kv : of_doc) rounds = std::max(rounds, kv.second.size());
    std::vector<XDoc> xd;
    for (size_t r = 0; r < rounds; r++) {
        std::vector<const i32*> slot_key(b->n.peers, nullptr);   // peer slot -> its part of the round's key
        std::vector<u8> h_req(b->n_docs, 0);
        bool cuts = false;
        for (const auto& kv : of_doc) {
            if (r >= kv.second.size()) continue;
            const Version& v = versions[kv.second[r]];
            const DocPeer* dp = &b->dpeer[b->peer_base[v.doc]];
            const i32* k = v.key.data();
            for (u32 p = 0; p < b->docs[v.doc].P; p++) {
                slot_key[b->docs[v.doc].peer0 + p] = k;
                for (i32 q = 0; q < k[0]; q++) cuts |= k[2 + 3 * q] < dp[p].end_counter;
                k += 1 + 3 * k[0];
            }
            h_req[v.doc] = 1;
        }
        std::vector<u32> h_span0(b->n.peers + 1, 0);
        std::vector<XSpan> h_spans;
        for (size_t slot = 0; slot < b->n.peers; slot++) {
            h_span0[slot] = (u32)h_spans.size();
            if (const i32* k = slot_key[slot])
                for (i32 q = 0; q < k[0]; q++) h_spans.push_back(XSpan{k[1 + 3 * q], k[2 + 3 * q], (u32)k[3 + 3 * q], 0});
        }
        h_span0[b->n.peers] = (u32)h_spans.size();
        e.bufs.push_back(export_round(b, h_span0, h_spans, cuts, h_req, xd));
        const uint8_t* blobs = e.bufs.back().get();
        for (size_t i = 0; i < n; i++) {
            if (version_of[i] == ~0u || versions[version_of[i]].round != r) continue;
            const XDoc& x = xd[doc_of(i)];
            if ((x.flags & 1) || x.exp_len == 0) e.answers[i] = lb_exports::Answer{LB_ERR_UNSUPPORTED, ERR_NOT_COVERED, nullptr, 0};
            else e.answers[i] = lb_exports::Answer{LB_OK, nullptr, blobs + x.exp_off, x.exp_len};
        }
    }
}

// Answers every request of lb_batch_export_updates (the arguments are checked): export(ExportMode::updates(from)) is
// one span [from, vv) per peer (change_store.rs:494-528); the last span given for a peer wins, peers the document lacks
// are ignored.
void export_requests(lb_batch* b, const lb_export_request* reqs, size_t n, lb_exports& e) {
    export_span_sets(b, n, [&](size_t i) { return reqs[i].doc; },
                     [&](size_t i, const DocInfo& di, const DocPeer* dp, SpanKey& key) -> const char* {
        std::vector<i32> h(di.P, 0);
        for (size_t k = 0; k < reqs[i].n_from; k++)
            for (u32 p = 0; p < di.P; p++)
                if (dp[p].id == reqs[i].from[k].peer) h[p] = reqs[i].from[k].end;
        for (u32 p = 0; p < di.P; p++) {
            const i32 start = std::max(h[p], 0);
            if (start < dp[p].end_counter) key.insert(key.end(), {1, start, dp[p].end_counter, 1});
            else key.push_back(0);
        }
        return nullptr;
    }, e);
}

// Answers every request of lb_batch_export_updates_in_range (the arguments are checked), as export_blocks_in_range takes
// its spans (change_store.rs:179-199): each is normalised (span.rs:51-68: a reversed span covers end+1 .. start+1); one
// that is empty, starts below 0 (iter_blocks then finds another peer's block), or names a peer the document lacks selects
// nothing; the others are clamped to the oplog vv.  In request order, a span continues the block of an earlier-listed
// span of its peer that ends exactly at its start (insert_change: the previous block by id), and starts a fresh block when
// no earlier-listed span of its peer lies below it.  The span sets the reference panics on or stores twice are refused.
void export_range_requests(lb_batch* b, const lb_range_request* reqs, size_t n, lb_exports& e) {
    export_span_sets(b, n, [&](size_t i) { return reqs[i].doc; },
                     [&](size_t i, const DocInfo& di, const DocPeer* dp, SpanKey& key) -> const char* {
        std::vector<std::vector<XSpan>> per(di.P);   // selected spans of each peer, in request order
        for (size_t k = 0; k < reqs[i].n_spans; k++) {
            const lb_id_span& sp = reqs[i].spans[k];
            u32 p = 0;
            while (p < di.P && dp[p].id != sp.peer) p++;
            if (p == di.P) continue;
            i64 s = sp.start, en = sp.end;
            if (en < s) { const i64 s2 = en + 1; en = s + 1; s = s2; }
            if (s < 0 || s == en) continue;
            en = std::min<i64>(en, dp[p].end_counter);
            if (s >= en) continue;
            per[p].push_back(XSpan{(i32)s, (i32)en, 1, (u32)per[p].size()});   // pad: the place in request order
        }
        for (u32 p = 0; p < di.P; p++) {
            // sorted by start, a span's neighbour below is the only candidate for the block it continues: one listed
            // earlier must end exactly at its start; one listed later leaves it a fresh block unless some span below it
            // was listed earlier still (that one ends below the neighbour's start: a gap)
            std::vector<XSpan>& v = per[p];
            std::sort(v.begin(), v.end(), [](const XSpan& x, const XSpan& y) { return x.start < y.start; });
            u32 first_below = ~0u;   // the earliest request place among the spans below the current one
            for (size_t a = 0; a < v.size(); a++) {
                if (a && v[a - 1].end > v[a].start) return ERR_SPANS_OVERLAP;
                if (a && v[a - 1].pad < v[a].pad) {
                    if (v[a - 1].end != v[a].start) return ERR_SPANS_GAP;
                    v[a].fresh = 0;
                } else if (first_below < v[a].pad) return ERR_SPANS_GAP;
                first_below = std::min(first_below, v[a].pad);
            }
            key.push_back((i32)v.size());
            for (const XSpan& x : v) key.insert(key.end(), {x.start, x.end, (i32)x.fresh});
        }
        return nullptr;
    }, e);
}

// Device bytes of JSON one writing pass produces at most (LB_JSON_STAGE_CAP overrides it, for testing: small chunks).
// A request larger than this is written alone, in a chunk of its own size.
u64 json_stage_cap() {
    const char* e = getenv("LB_JSON_STAGE_CAP");
    return e ? std::max<u64>(strtoull(e, nullptr, 10), 1) : (256ull << 20);
}

// Answers every request of lb_batch_export_json_updates (the arguments are checked) in one device pass: the import
// store of every named document is rebuilt once (k_jx_store; it does not depend on any version), a thread per request
// orders and lists its output changes (k_jx_order), a thread per output change counts its bytes (k_jx_changes), the host
// scans the sizes and places the requests, and the changes and envelopes are written chunk by chunk, each chunk at most
// json_stage_cap() bytes.  Each version becomes the request's refined vectors over the document's peer slots
// (json_schema.rs:31-45: a peer the document lacks contributes nothing, counters are clamped to the oplog vv).
void json_requests(lb_batch* b, const lb_json_request* reqs, size_t n, lb_exports& e) {
    e.answers.assign(n, lb_exports::Answer{LB_OK, nullptr, nullptr, 0});
    const u32 D = (u32)b->n_docs;
    std::vector<JxReq> jr;
    std::vector<size_t> of;            // device request -> request
    std::vector<i32> h_start, h_end;
    std::vector<u8> h_req(D, 0);
    for (size_t i = 0; i < n; i++) {
        const size_t doc = reqs[i].doc;
        const DocInfo& di = b->docs[doc];
        if (di.code != DOC_OK) { e.answers[i] = doc_error(di); continue; }
        const DocPeer* dp = &b->dpeer[b->peer_base[doc]];
        auto refine = [&](const lb_id_span* v, size_t nv, std::vector<i32>& out) {
            const size_t base = out.size();
            out.resize(base + di.P, 0);
            for (size_t k = 0; k < nv; k++)   // the last span for a peer wins
                for (u32 p = 0; p < di.P; p++)
                    if (dp[p].id == v[k].peer) out[base + p] = std::max(0, std::min(v[k].end, dp[p].end_counter));
        };
        refine(reqs[i].start, reqs[i].n_start, h_start);
        refine(reqs[i].end, reqs[i].n_end, h_end);
        JxReq r{};
        r.doc = (u32)doc;
        r.flags = reqs[i].flags & JX_NO_PEER_COMPRESSION;
        r.slot0 = h_start.size() - di.P;
        jr.push_back(r);
        of.push_back(i);
        h_req[doc] = 1;
    }
    if (jr.empty()) return;
    Dev& dv = b->dev;
    cudaStream_t st = dv.stream;
    const u64 NR = jr.size(), S = std::max<size_t>(h_start.size(), 1);
    JxReq* d_jr = dv.alloc<JxReq>(NR);
    JxScratch s{dv.alloc<i32>(S), dv.alloc<i32>(S), dv.alloc<u32>(S), dv.alloc<u32>(S), dv.alloc<u32>(S)};
    u32* d_pf0 = dv.alloc<u32>(b->n.peers + 1);
    u32* d_pfn = dv.alloc<u32>(b->n.peers + 1);
    CK(cudaMemcpyAsync(s.start, h_start.data(), sizeof(i32) * h_start.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(s.end, h_end.data(), sizeof(i32) * h_end.size(), cudaMemcpyHostToDevice, st));
    BatchTables xt = export_pass(b, h_req);
    LB_BATCH_LAUNCH(b, k_jx_store, nblk(D, 64), 64, 0, b->d_docs, D, xt, d_pf0, d_pfn);
    // every request gets as many output slots as its document has stored changes
    std::vector<XDoc> xd(D);
    CK(cudaMemcpyAsync(xd.data(), xt.xdoc, sizeof(XDoc) * D, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    trace_point(b, "json: import store");
    u64 slots = 0;
    for (JxReq& r : jr) { r.ch0 = slots; slots += (xd[r.doc].flags & 1) ? 0 : xd[r.doc].n_fc; }
    u32* d_och = dv.alloc<u32>(std::max<u64>(slots, 1));
    CK(cudaMemcpyAsync(d_jr, jr.data(), sizeof(JxReq) * NR, cudaMemcpyHostToDevice, st));
    LB_BATCH_LAUNCH(b, k_jx_order, nblk(NR, 64), 64, 0, b->d_docs, xt, d_jr, (u32)NR, s, d_pf0, d_pfn, d_och);
    CK(cudaMemcpyAsync(jr.data(), d_jr, sizeof(JxReq) * NR, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    trace_point(b, "json: order");
    // the output changes of all requests, numbered consecutively; a thread per change counts its bytes
    u64 NOUT = 0;
    for (JxReq& r : jr) { r.c0 = NOUT; NOUT += r.n_out; }
    std::vector<u32> h_oreq(std::max<u64>(NOUT, 1));
    for (u64 r = 0; r < NR; r++) std::fill(h_oreq.begin() + jr[r].c0, h_oreq.begin() + jr[r].c0 + jr[r].n_out, (u32)r);
    u32* d_oreq = dv.alloc<u32>(h_oreq.size());
    u32* d_olen = dv.alloc<u32>(h_oreq.size());
    u64* d_ooff = dv.alloc<u64>(h_oreq.size());
    CK(cudaMemcpyAsync(d_jr, jr.data(), sizeof(JxReq) * NR, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_oreq, h_oreq.data(), sizeof(u32) * h_oreq.size(), cudaMemcpyHostToDevice, st));
    std::vector<u32> h_olen(h_oreq.size(), 0);
    if (NOUT) {
        LB_BATCH_LAUNCH(b, k_jx_changes, nblk(NOUT, 64), 64, 0, b->d_docs, xt, d_jr, s, d_pf0, d_pfn, d_och, d_oreq, 0ull, NOUT,
                        d_olen, (const u64*)nullptr, (u8*)nullptr, 0ull);
        CK(cudaMemcpyAsync(h_olen.data(), d_olen, sizeof(u32) * NOUT, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    trace_point(b, "json: count");
    // place the requests and their changes: envelope head, the changes, "]}"
    std::vector<u64> h_ooff(h_oreq.size(), 0);
    u64 total = 0;
    for (JxReq& r : jr) {
        r.off = total;
        if (r.len == JX_UNSUPPORTED) continue;
        u64 w = total + r.pre_len;
        for (u64 k = r.c0; k < r.c0 + r.n_out; k++) { h_ooff[k] = w; w += h_olen[k]; }
        r.len = w + 2 - total;
        total += r.len;
    }
    CK(cudaMemcpyAsync(d_jr, jr.data(), sizeof(JxReq) * NR, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_ooff, h_ooff.data(), sizeof(u64) * h_ooff.size(), cudaMemcpyHostToDevice, st));
    e.bufs.emplace_back(new uint8_t[total + 1]);
    uint8_t* host = e.bufs.back().get();
    const u64 cap = json_stage_cap();
    u8* d_out = nullptr;
    u64 d_out_cap = 0;
    for (u64 r0 = 0; r0 < NR;) {
        u64 r1 = r0, bytes = 0;
        while (r1 < NR) {
            const u64 len = jr[r1].len == JX_UNSUPPORTED ? 0 : jr[r1].len;
            if (r1 > r0 && bytes + len > cap) break;
            bytes += len;
            r1++;
        }
        if (bytes > d_out_cap) {
            if (d_out) dv.release(d_out);
            d_out = dv.alloc<u8>(bytes);
            d_out_cap = bytes;
        }
        const u64 base = jr[r0].off, k0 = jr[r0].c0, k1 = jr[r1 - 1].c0 + jr[r1 - 1].n_out;
        if (k1 > k0)
            LB_BATCH_LAUNCH(b, k_jx_changes, nblk(k1 - k0, 64), 64, 0, b->d_docs, xt, d_jr, s, d_pf0, d_pfn, d_och, d_oreq, k0, k1,
                            (u32*)nullptr, d_ooff, d_out, base);
        LB_BATCH_LAUNCH(b, k_jx_envelope, nblk(r1 - r0, 64), 64, 0, b->d_docs, xt, d_jr, (u32)r0, (u32)r1, s, d_pf0, d_pfn,
                        d_out, base);
        if (bytes && !lbstage::download(d_out, host + base, bytes, st)) { g_last_error = "json d2h failed"; throw lb_status(LB_ERR_CUDA); }
        CK(cudaStreamSynchronize(st));
        r0 = r1;
    }
    trace_point(b, "json: write");
    for (u64 k = 0; k < NR; k++) {
        if (jr[k].len == JX_UNSUPPORTED) e.answers[of[k]] = lb_exports::Answer{LB_ERR_UNSUPPORTED, ERR_NOT_COVERED, nullptr, 0};
        else e.answers[of[k]] = lb_exports::Answer{LB_OK, nullptr, host + jr[k].off, (size_t)jr[k].len};
    }
    if (d_out) dv.release(d_out);
    dv.release(xt.x_req); dv.release(d_jr); dv.release(s.start); dv.release(s.end); dv.release(s.reg); dv.release(s.ord);
    dv.release(s.cur); dv.release(d_pf0); dv.release(d_pfn); dv.release(xt.xdoc); dv.release(d_och); dv.release(d_oreq);
    dv.release(d_olen); dv.release(d_ooff);
}

// The body of the lb_batch_export_* calls: the batch and every request are checked before anything launches (a request's
// document index, then refused(request): why its pointers are bad, or nullptr), then answer() fills one answer per
// request under the batch's export lock.
template <class Req, class Refused>
lb_status export_call(const lb_batch* cb, const Req* reqs, size_t n_reqs, lb_exports** out, Refused refused,
                      void (*answer)(lb_batch*, const Req*, size_t, lb_exports&)) {
    lb_batch* b = const_cast<lb_batch*>(cb);
    if (!b || !out || (!reqs && n_reqs)) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    *out = nullptr;
    if (!(b->flags & LB_FLAG_EXPORT)) { g_last_error = "batch was imported without LB_FLAG_EXPORT"; return LB_ERR_INVALID_ARG; }
    for (size_t i = 0; i < n_reqs; i++) {
        if (reqs[i].doc >= b->n_docs) { g_last_error = "document index out of range"; return LB_ERR_INVALID_ARG; }
        if (const char* err = refused(reqs[i])) { g_last_error = err; return LB_ERR_INVALID_ARG; }
    }
    std::unique_ptr<lb_exports> e(new lb_exports());
    std::lock_guard<std::mutex> g(b->export_mu);
    try {
        answer(b, reqs, n_reqs, *e);
    } catch (lb_status s) {
        return s;
    }
    *out = e.release();
    return LB_OK;
}

}  // namespace

// After an import into a docset: every document of the batch whose import succeeded gets its new stored form -- the
// blobs it was built from (earlier ones first), copied out of the batch's byte buffer, or, with LB_FLAG_COMPACT, the
// blob it re-exports (ExportMode::all_updates) when nothing is pending and the export phase covers it.  A document
// whose import failed (checksum, decode, ...) keeps its earlier state: the reference rejects such an import before any
// state change.
void docset_store(lb_docset* set, lb_batch* b, const std::vector<u64>& offs, const std::vector<u32>& lens) {
    const size_t nd = b->n_docs;
    struct Pick { size_t doc; bool exported; };
    std::vector<Pick> picks;
    u64 total = 0;
    for (size_t d = 0; d < nd; d++) {
        const DocInfo& di = b->docs[d];
        if (di.code != DOC_OK && di.code != DOC_ERR_UNSUPPORTED) continue;
        // LB_FLAG_COMPACT: the document is replaced by a fresh one that imported its own export (what a host does to drop
        // redundant history: `fresh.import(doc.export(all_updates))`); otherwise it keeps every blob it ever imported, in
        // order, so that a later export is byte-identical to the reference's after the same sequence of imports (the
        // op segmentation of an export depends on which blob brought which piece of a change)
        bool exported = (b->flags & LB_FLAG_COMPACT) && di.code == DOC_OK && di.n_pending == 0 && d < b->xdocs.size() &&
                        !(b->xdocs[d].flags & 1) && b->xdocs[d].exp_len > 0;
        picks.push_back(Pick{d, exported});
        if (exported) total += ((u64)b->xdocs[d].exp_len + 15) & ~(u64)15;
        else for (u32 q = b->doc_blob0[d]; q < b->doc_blob0[d + 1]; q++) total += ((u64)lens[q] + 15) & ~(u64)15;
    }
    if (picks.empty()) return;
    auto buf = std::make_shared<DocsetBuf>();
    buf->bytes = total + 64;
    if (cudaMalloc((void**)&buf->d, buf->bytes) != cudaSuccess) {
        cudaGetLastError();
        g_last_error = "docset: out of device memory for the stored documents";
        throw lb_status(LB_ERR_OOM);
    }
    std::vector<CopySeg> segs;
    std::vector<std::pair<u64, DocsetDoc>> fresh;
    u64 w = 0;
    for (const Pick& pk : picks) {
        DocsetDoc nd_;
        auto push = [&](const u8* src, u32 len) {
            segs.push_back(CopySeg{src, buf->d + w, len});
            nd_.blobs.push_back(DocsetBlob{buf, w, len});
            w += ((u64)len + 15) & ~(u64)15;
        };
        if (pk.exported) push(b->exported.d + b->xdocs[pk.doc].exp_off, b->xdocs[pk.doc].exp_len);
        else for (u32 q = b->doc_blob0[pk.doc]; q < b->doc_blob0[pk.doc + 1]; q++) push(b->tb.bytes + offs[q], lens[q]);
        fresh.push_back({b->doc_ids[pk.doc], std::move(nd_)});
    }
    CopySeg* d_segs = b->dev.alloc<CopySeg>(segs.size());
    CK(cudaMemcpyAsync(d_segs, segs.data(), sizeof(CopySeg) * segs.size(), cudaMemcpyHostToDevice, b->dev.stream));
    LB_BATCH_LAUNCH(b, k_copy_segments, nblk((u64)segs.size() * 32, 128), 128, 0, d_segs, (u32)segs.size());
    CK(cudaStreamSynchronize(b->dev.stream));
    for (auto& kv : fresh) {
        DocsetDoc& slot = set->docs[kv.first];
        for (const DocsetBlob& ob : slot.blobs) set->stored_bytes -= ob.len;
        slot = std::move(kv.second);
        for (const DocsetBlob& nb : slot.blobs) set->stored_bytes += nb.len;
    }
}

// The host-buffer entry points (they share import_host).
enum class HostEntry { IMPORT, IMPORT_AT, DOCSET_IMPORT, DOCSET_CHECKOUT, DOCSET_READ };

extern "C" {

// Host-buffer import, shared by lb_import_batch (fresh documents), lb_docset_import (documents with an earlier state:
// their stored blobs come first, already in device memory, and count as `n_prior` for the import status) and the
// checkout entry points: `at` names the documents built at an earlier version (k_checkout.cuh).  For DOCSET_CHECKOUT the
// documents are the requests themselves, one per entry of `at`, each made of its document's stored blobs only; for
// DOCSET_READ they are the listed `read_ids`, each made of its stored blobs, at the latest version and exported.  In both
// the docset is read, never written.
// The flags each entry point takes are decided here: a checked-out document answers no cursor and is not exported, a
// read writes nothing back, and a docset import or read is always exported (the re-export is what a stored document
// keeps, and what a read answers from).  The cursor flag is refused before a null argument, the other flags after it.
static lb_status import_host(HostEntry entry, lb_docset* set, const lb_blob* blobs, size_t n_blobs, const lb_version* at,
                             size_t n_at, const uint64_t* read_ids, size_t n_read, const lb_options* opt, lb_batch** out) {
    const bool checkout = entry == HostEntry::IMPORT_AT || entry == HostEntry::DOCSET_CHECKOUT;
    lb_options o2 = opt ? *opt : lb_options{};
    if (checkout && (o2.flags & LB_FLAG_CURSORS)) { g_last_error = "cursors are not answered on checked-out documents"; return LB_ERR_INVALID_ARG; }
    if (!out || (!blobs && n_blobs) || (!at && n_at) || (!read_ids && n_read)) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    *out = nullptr;
    if (checkout) {
        if (o2.flags & (LB_FLAG_EXPORT | LB_FLAG_COMPACT)) {
            g_last_error = "a checked-out document is not exported (LB_FLAG_EXPORT / LB_FLAG_COMPACT)";
            return LB_ERR_INVALID_ARG;
        }
        for (size_t i = 0; i < n_at; i++)
            if (!at[i].frontiers && at[i].n_frontiers) { g_last_error = "null frontiers"; return LB_ERR_INVALID_ARG; }
    }
    if (entry == HostEntry::DOCSET_READ && (o2.flags & LB_FLAG_COMPACT)) { g_last_error = "LB_FLAG_COMPACT on a read: the docset is not written"; return LB_ERR_INVALID_ARG; }
    if (set) o2.device = set->device;
    if (entry == HostEntry::DOCSET_IMPORT || entry == HostEntry::DOCSET_READ) o2.flags |= LB_FLAG_EXPORT;
    return import_with_new_batch(&o2, out, [&](lb_batch* b) {
        if (n_blobs >= 0x7FFFFFFFull) { g_last_error = "too many blobs"; throw lb_status(LB_ERR_INVALID_ARG); }
        b->eager_json = true;   // host buffers in, host results expected
        // blobs with the same doc_id form one document (LoroDoc::import_batch); documents are numbered in order of
        // first appearance and their blobs laid out consecutively, in the order given
        std::vector<u32> order(n_blobs);
        std::vector<u32> count;   // new blobs per document
        std::unordered_map<u64, u32> doc_of;
        std::vector<u32> doc_idx(n_blobs);
        for (size_t i = 0; i < n_blobs; i++) {
            auto it = doc_of.find(blobs[i].doc_id);
            if (it == doc_of.end()) {
                it = doc_of.emplace(blobs[i].doc_id, (u32)count.size()).first;
                count.push_back(0);
                b->doc_ids.push_back(blobs[i].doc_id);
            }
            doc_idx[i] = it->second;
            count[it->second]++;
        }
        size_t nd = count.size();
        std::vector<u32> first(nd + 1, 0);
        for (size_t d = 0; d < nd; d++) first[d + 1] = first[d] + count[d];
        std::vector<u32> cursor(first.begin(), first.end() - 1);
        for (size_t i = 0; i < n_blobs; i++) order[cursor[doc_idx[i]]++] = (u32)i;
        // import_batch imports its blobs sorted by (mode, number of changes descending), stably
        // (loro.rs:1194-1202): the order decides where payloads land in the document's arenas, which the
        // re-export merge rules look at
        for (size_t d = 0; d < nd; d++) {
            u32 q0 = first[d], q1 = first[d + 1];
            if (q1 - q0 < 2) continue;
            std::vector<std::pair<std::pair<u32, i64>, u32>> keyed;
            for (u32 q = q0; q < q1; q++) {
                const lb_blob& bl = blobs[order[q]];
                keyed.push_back({{blob_mode(bl.ptr, bl.len), -(i64)blob_change_count(bl.ptr, bl.len)}, order[q]});
            }
            std::stable_sort(keyed.begin(), keyed.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
            for (u32 q = q0; q < q1; q++) order[q] = keyed[q - q0].second;
        }
        if (entry == HostEntry::DOCSET_CHECKOUT)   // one document per request, in request order (no new blobs)
            for (size_t i = 0; i < n_at; i++) { b->doc_ids.push_back(at[i].doc_id); count.push_back(0); nd++; }
        for (size_t i = 0; i < n_read; i++) {   // one document per listed id, in list order (no new blobs)
            if (!doc_of.emplace(read_ids[i], (u32)nd).second) { g_last_error = "doc_id listed twice"; throw lb_status(LB_ERR_INVALID_ARG); }
            b->doc_ids.push_back(read_ids[i]); count.push_back(0); nd++;
        }
        b->stored_only = entry == HostEntry::DOCSET_CHECKOUT || entry == HostEntry::DOCSET_READ;
        b->n_docs = nd;
        if (checkout) {
            b->ck_range.assign(2 * nd, CK_LATEST);
            for (size_t i = 0; i < n_at; i++) {
                u32 d = (u32)i;
                if (entry == HostEntry::IMPORT_AT) {
                    auto it = doc_of.find(at[i].doc_id);
                    if (it == doc_of.end()) { g_last_error = "checkout of a doc_id no blob carries"; throw lb_status(LB_ERR_INVALID_ARG); }
                    d = it->second;
                    if (b->ck_range[2 * d] != CK_LATEST) { g_last_error = "doc_id requested twice"; throw lb_status(LB_ERR_INVALID_ARG); }
                }
                b->ck_range[2 * d] = (u32)b->ck_peer.size();
                for (size_t k = 0; k < at[i].n_frontiers; k++) {   // one span [counter, counter + 1) per id
                    b->ck_peer.push_back(at[i].frontiers[k].peer);
                    b->ck_ctr.push_back(at[i].frontiers[k].start);
                }
                b->ck_range[2 * d + 1] = (u32)b->ck_peer.size();
            }
            if (b->ck_peer.size() >= CK_LATEST) { g_last_error = "too many frontier ids"; throw lb_status(LB_ERR_INVALID_ARG); }
        }
        // the blob list of the batch: per document, its stored blobs (device) then the new ones (host)
        std::vector<DocsetDoc*> prior(nd, nullptr);
        size_t n_prior_total = 0;
        if (set) {
            b->doc_nprior.assign(nd, 0);
            for (size_t d = 0; d < nd; d++) {
                auto it = set->docs.find(b->doc_ids[d]);
                if (it == set->docs.end()) continue;
                prior[d] = &it->second;
                b->doc_nprior[d] = (u32)it->second.blobs.size();
                n_prior_total += it->second.blobs.size();
            }
        }
        const size_t Q = n_blobs + n_prior_total;
        if (Q >= 0x7FFFFFFFull) { g_last_error = "too many blobs"; throw lb_status(LB_ERR_INVALID_ARG); }
        b->n_blobs = Q;
        b->doc_blob0.assign(nd + 1, 0);
        b->blob_doc.resize(Q);
        std::vector<u64> offs(Q + 1);
        std::vector<u32> lens(Q + 1, 0);
        std::vector<lbstage::BlobView> views;      // host blobs, with their offsets in the batch buffer
        std::vector<u64> view_offs;
        std::vector<CopySeg> segs;                 // stored blobs: device-to-device (dst filled in below)
        std::vector<u64> seg_offs;
        views.reserve(n_blobs);
        view_offs.reserve(n_blobs + 1);
        // the host blobs fill [0, H) of the batch buffer in one contiguous upload, the stored blobs follow
        u64 total = 0, ptotal = 0;
        for (size_t i = 0; i < n_blobs; i++) ptotal += (blobs[i].len + 15) & ~(u64)15;
        size_t q = 0, hq = 0;
        for (size_t d = 0; d < nd; d++) {
            b->doc_blob0[d] = (u32)q;
            auto place = [&](u64& w, u64 len) {   // blob q of document d at byte w of the batch buffer
                offs[q] = w;
                lens[q] = (u32)len;
                b->blob_doc[q++] = (u32)d;
                w += (len + 15) & ~(u64)15;
                b->counters.blob_bytes += len;
            };
            if (prior[d])
                for (const DocsetBlob& sb : prior[d]->blobs) {
                    segs.push_back(CopySeg{sb.buf->d + sb.off, nullptr, sb.len});
                    seg_offs.push_back(ptotal);
                    place(ptotal, sb.len);
                }
            for (u32 k = 0; k < count[d]; k++, hq++) {
                const lb_blob& bl = blobs[order[hq]];
                if (bl.len > 0xFFFFFFF0ull || (!bl.ptr && bl.len)) {
                    g_last_error = "blob too large or null";
                    throw lb_status(LB_ERR_INVALID_ARG);
                }
                views.push_back(lbstage::BlobView{bl.ptr, bl.len});
                view_offs.push_back(total);
                place(total, bl.len);
            }
        }
        b->doc_blob0[nd] = (u32)q;
        offs[Q] = ptotal;
        view_offs.push_back(total);
        total = ptotal;
        // stage through the pinned ring: host gather of slot k overlaps the DMA of slot k-1 (host_stage.hpp)
        mark(b, EV_START);
        u8* d_bytes = b->dev.alloc<u8>(total + 64);
        if (!segs.empty()) {
            for (size_t k = 0; k < segs.size(); k++) segs[k].dst = d_bytes + seg_offs[k];
            CopySeg* d_segs = b->dev.alloc<CopySeg>(segs.size());
            CK(cudaMemcpyAsync(d_segs, segs.data(), sizeof(CopySeg) * segs.size(), cudaMemcpyHostToDevice, b->dev.stream));
            LB_BATCH_LAUNCH(b, k_copy_segments, nblk((u64)segs.size() * 32, 128), 128, 0, d_segs, (u32)segs.size());
            CK(cudaStreamSynchronize(b->dev.stream));   // `segs` is pageable host memory
        }
        if (!views.empty() && !lbstage::upload_blobs(views.data(), view_offs.data(), views.size(), d_bytes, b->dev.stream)) {
            g_last_error = "h2d staging failed";
            throw lb_status(LB_ERR_CUDA);
        }
        lb_status s = upload_and_run(b, offs, lens, d_bytes);
        CK(cudaStreamSynchronize(b->dev.stream));
        if (s == LB_OK && set && !b->stored_only) docset_store(set, b, offs, lens);
        return s;
    });
}

lb_status lb_import_batch(const lb_blob* blobs, size_t n_blobs, const lb_options* opt, lb_batch** out) {
    return import_host(HostEntry::IMPORT, nullptr, blobs, n_blobs, nullptr, 0, nullptr, 0, opt, out);
}

lb_status lb_import_batch_at(const lb_blob* blobs, size_t n_blobs, const lb_version* at, size_t n_at, const lb_options* opt,
                             lb_batch** out) {
    return import_host(HostEntry::IMPORT_AT, nullptr, blobs, n_blobs, at, n_at, nullptr, 0, opt, out);
}

lb_status lb_docset_new(const lb_options* opt, lb_docset** out) {
    if (!out) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    *out = nullptr;
    lb_status s = check_device(opt);
    if (s != LB_OK) return s;
    lb_docset* set = new lb_docset();
    set->device = opt ? opt->device : 0;
    *out = set;
    return LB_OK;
}

void lb_docset_free(lb_docset* set) { delete set; }

size_t lb_docset_doc_count(const lb_docset* set) { return set ? set->docs.size() : 0; }

uint64_t lb_docset_stored_bytes(const lb_docset* set) { return set ? set->stored_bytes : 0; }

lb_status lb_docset_import(lb_docset* set, const lb_blob* blobs, size_t n_blobs, const lb_options* opt, lb_batch** out) {
    if (!set) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> g(set->mu);
    return import_host(HostEntry::DOCSET_IMPORT, set, blobs, n_blobs, nullptr, 0, nullptr, 0, opt, out);
}

lb_status lb_docset_checkout(lb_docset* set, const lb_version* at, size_t n_at, const lb_options* opt, lb_batch** out) {
    if (!set) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> g(set->mu);
    return import_host(HostEntry::DOCSET_CHECKOUT, set, nullptr, 0, at, n_at, nullptr, 0, opt, out);
}

lb_status lb_docset_read(lb_docset* set, const uint64_t* doc_ids, size_t n, const lb_options* opt, lb_batch** out) {
    if (!set) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> g(set->mu);
    return import_host(HostEntry::DOCSET_READ, set, nullptr, 0, nullptr, 0, doc_ids, n, opt, out);
}

lb_status lb_import_batch_device(const uint8_t* d_bytes, const uint64_t* offsets, const uint32_t* blob_lens,
                                 size_t n_docs, const lb_options* opt, lb_batch** out) {
    if (!out || ((!offsets || !blob_lens || !d_bytes) && n_docs)) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    *out = nullptr;
    return import_with_new_batch(opt, out, [&](lb_batch* b) {
        b->n_docs = n_docs;
        std::vector<u64> offs(n_docs + 1);
        std::vector<u32> lens(n_docs + 1, 0);
        for (size_t i = 0; i < n_docs; i++) {
            if (offsets[i] & 15) { g_last_error = "blob offsets must be multiples of 16"; throw lb_status(LB_ERR_INVALID_ARG); }
            offs[i] = offsets[i];
            lens[i] = blob_lens[i];
            b->doc_ids.push_back(i);
            b->blob_doc.push_back((u32)i);
            b->doc_blob0.push_back((u32)i);
            b->counters.blob_bytes += lens[i];
        }
        offs[n_docs] = n_docs ? offsets[n_docs - 1] + lens[n_docs - 1] : 0;
        b->doc_blob0.push_back((u32)n_docs);
        b->n_blobs = n_docs;
        mark(b, EV_START);
        return upload_and_run(b, offs, lens, d_bytes);
    });
}

size_t lb_doc_count(const lb_batch* b) { return b ? b->n_docs : 0; }

lb_status lb_doc_status(const lb_batch* b, size_t doc, lb_import_status* out) {
    if (!b || !out || doc >= b->n_docs) { g_last_error = "bad argument"; return LB_ERR_INVALID_ARG; }
    out->code = (lb_doc_code)b->docs[doc].code;
    out->n_success = b->span_off[0][doc + 1] - b->span_off[0][doc];
    out->success = b->spans[0].data() + b->span_off[0][doc];
    out->n_pending = b->span_off[1][doc + 1] - b->span_off[1][doc];
    out->pending = b->spans[1].data() + b->span_off[1][doc];
    return LB_OK;
}

// document doc's spans of kind k (b->spans: 2 the vv, 3 the frontiers)
static lb_status doc_spans(const lb_batch* b, int k, size_t doc, const lb_id_span** spans, size_t* n) {
    if (!b || !spans || !n || doc >= b->n_docs) { g_last_error = "bad argument"; return LB_ERR_INVALID_ARG; }
    *spans = b->spans[k].data() + b->span_off[k][doc];
    *n = b->span_off[k][doc + 1] - b->span_off[k][doc];
    return LB_OK;
}
lb_status lb_doc_vv(const lb_batch* b, size_t doc, const lb_id_span** spans, size_t* n) { return doc_spans(b, 2, doc, spans, n); }
lb_status lb_doc_frontiers(const lb_batch* b, size_t doc, const lb_id_span** spans, size_t* n) { return doc_spans(b, 3, doc, spans, n); }

lb_status lb_doc_json(const lb_batch* cb, size_t doc, const char** utf8, size_t* len) {
    lb_batch* b = const_cast<lb_batch*>(cb);
    if (!b || !utf8 || !len || doc >= b->n_docs) { g_last_error = "bad argument"; return LB_ERR_INVALID_ARG; }
    if (b->flags & LB_FLAG_NO_JSON) { g_last_error = "batch was imported with LB_FLAG_NO_JSON"; return LB_ERR_INVALID_ARG; }
    if (b->json_thread.joinable()) {
        b->json_thread.join();
        if (!b->json_ok) { g_last_error = "json d2h failed"; return LB_ERR_CUDA; }
    }
    if (lb_status s = b->json.fetch(b->dev.stream, "json d2h failed")) return s;
    const DocInfo& di = b->docs[doc];
    if (di.code != DOC_OK) { *utf8 = ""; *len = 0; return LB_OK; }
    *utf8 = b->json.host + di.json_off;
    *len = di.json_len;
    return LB_OK;
}

lb_status lb_doc_attribution(const lb_batch* cb, size_t doc, const char** utf8, size_t* len) {
    lb_batch* b = const_cast<lb_batch*>(cb);
    if (!b || !utf8 || !len || doc >= b->n_docs) { g_last_error = "bad argument"; return LB_ERR_INVALID_ARG; }
    if (!(b->flags & LB_FLAG_ATTRIBUTION)) { g_last_error = "batch was imported without LB_FLAG_ATTRIBUTION"; return LB_ERR_INVALID_ARG; }
    if (!b->attr.fetched) {   // the offsets, then the text: one download of each
        b->attr_off.assign(b->n_docs + 1, 0);
        if (cudaMemcpy(b->attr_off.data(), b->d_attr_off, sizeof(u64) * (b->n_docs + 1), cudaMemcpyDeviceToHost) != cudaSuccess) {
            g_last_error = "attribution d2h failed";
            return LB_ERR_CUDA;
        }
    }
    if (lb_status s = b->attr.fetch(b->dev.stream, "attribution d2h failed")) return s;
    if (b->docs[doc].code != DOC_OK) { *utf8 = ""; *len = 0; return LB_OK; }
    *utf8 = b->attr.host + b->attr_off[doc];
    *len = b->attr_off[doc + 1] - b->attr_off[doc];
    return LB_OK;
}

lb_status lb_batch_cursor_pos(const lb_batch* cb, const lb_cursor* reqs, size_t n, lb_cursor_result* out) {
    lb_batch* b = const_cast<lb_batch*>(cb);
    if (!b || ((!reqs || !out) && n)) { g_last_error = "null argument"; return LB_ERR_INVALID_ARG; }
    if (!(b->flags & LB_FLAG_CURSORS)) { g_last_error = "batch was imported without LB_FLAG_CURSORS"; return LB_ERR_INVALID_ARG; }
    // the requests, then the root names they carry, packed for one upload
    size_t name_bytes = 0;
    for (size_t i = 0; i < n; i++) {
        if (reqs[i].doc >= b->n_docs) { g_last_error = "document index out of range"; return LB_ERR_INVALID_ARG; }
        if (reqs[i].is_root && !reqs[i].name && reqs[i].name_len) { g_last_error = "null root container name"; return LB_ERR_INVALID_ARG; }
        if (reqs[i].is_root) name_bytes += reqs[i].name_len;
    }
    if (!n) return LB_OK;
    const size_t req_bytes = sizeof(CurReq) * n;
    std::vector<u8> host(req_bytes + name_bytes);
    CurReq* hq = (CurReq*)host.data();
    size_t noff = 0;
    for (size_t i = 0; i < n; i++) {
        const lb_cursor& c = reqs[i];
        CurReq& q = hq[i];
        memset(&q, 0, sizeof(q));
        q.doc = c.doc;
        q.is_root = c.is_root ? 1 : 0;
        q.type = c.type;
        q.has_id = c.has_id ? 1 : 0;
        q.side = c.side;
        q.tpeer = c.id_peer;
        q.tctr = c.id_counter;
        if (q.is_root) {
            if (c.name_len >= 0xFFFFFFFFull) { g_last_error = "root container name too long"; return LB_ERR_INVALID_ARG; }
            q.name_off = noff;
            q.name_len = (u32)c.name_len;
            if (c.name_len) memcpy(host.data() + req_bytes + noff, c.name, c.name_len);
            noff += c.name_len;
        } else {
            q.cpeer = c.peer;
            q.ccounter = c.counter;
        }
    }
    std::lock_guard<std::mutex> g(b->export_mu);   // device work on demand runs one call at a time
    try {
        Dev& dv = b->dev;
        cudaStream_t st = b->dev.stream;
        u8* d_in = dv.alloc<u8>(host.size());
        lb_cursor_result* d_out = dv.alloc<lb_cursor_result>(n);
        CK(cudaMemcpyAsync(d_in, host.data(), host.size(), cudaMemcpyHostToDevice, st));
        LB_BATCH_LAUNCH(b, k_cursor_query, nblk((u64)n * 32, 128), 128, 0, b->d_docs, b->tb, b->cur, (const CurReq*)d_in,
                        (const u8*)(d_in + req_bytes), (u64)n, d_out);
        CK(cudaMemcpyAsync(out, d_out, sizeof(lb_cursor_result) * n, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        dv.release(d_in);
        dv.release(d_out);
    } catch (lb_status s) {
        return s;
    }
    return LB_OK;
}

lb_status lb_doc_export_updates(const lb_batch* cb, size_t doc, const lb_id_span* from, size_t n_from,
                                const uint8_t** bytes, size_t* len) {
    lb_batch* b = const_cast<lb_batch*>(cb);
    if (!b || !bytes || !len || doc >= b->n_docs) { g_last_error = "bad argument"; return LB_ERR_INVALID_ARG; }
    if (!(b->flags & LB_FLAG_EXPORT)) { g_last_error = "batch was imported without LB_FLAG_EXPORT"; return LB_ERR_INVALID_ARG; }
    if (b->docs[doc].code != DOC_OK) {
        lb_exports::Answer a = doc_error(b->docs[doc]);
        g_last_error = a.error;
        return a.status;
    }
    std::lock_guard<std::mutex> g(b->export_mu);
    if (from && n_from) {   // export(ExportMode::updates(from)): a one-request lb_batch_export_updates
        lb_export_request rq{doc, from, n_from};
        lb_exports e;
        try {
            export_requests(b, &rq, 1, e);
        } catch (lb_status s) {
            return s;
        }
        const lb_exports::Answer& a = e.answers[0];
        if (a.status != LB_OK) { g_last_error = a.error; return a.status; }
        std::vector<uint8_t>& buf = b->from_exports[doc];
        buf.assign(a.bytes, a.bytes + a.len);
        *bytes = buf.data();
        *len = buf.size();
        return LB_OK;
    }
    const XDoc& x = b->xdocs[doc];
    if ((x.flags & 1) || x.exp_len == 0) { g_last_error = ERR_NOT_COVERED; return LB_ERR_UNSUPPORTED; }
    if (lb_status s = b->exported.fetch(b->dev.stream, "export d2h failed")) return s;
    *bytes = (const uint8_t*)b->exported.host + x.exp_off;
    *len = x.exp_len;
    return LB_OK;
}

lb_status lb_batch_export_updates(const lb_batch* cb, const lb_export_request* reqs, size_t n_reqs, lb_exports** out) {
    return export_call(cb, reqs, n_reqs, out, [](const lb_export_request& r) -> const char* {
        return !r.from && r.n_from ? "null from with n_from > 0" : nullptr;
    }, export_requests);
}

lb_status lb_batch_export_updates_in_range(const lb_batch* cb, const lb_range_request* reqs, size_t n_reqs, lb_exports** out) {
    return export_call(cb, reqs, n_reqs, out, [](const lb_range_request& r) -> const char* {
        return !r.spans && r.n_spans ? "null spans with n_spans > 0" : nullptr;
    }, export_range_requests);
}

lb_status lb_batch_export_json_updates(const lb_batch* cb, const lb_json_request* reqs, size_t n_reqs, lb_exports** out) {
    return export_call(cb, reqs, n_reqs, out, [](const lb_json_request& r) -> const char* {
        return (!r.start && r.n_start) || (!r.end && r.n_end) ? "null version with a count > 0" : nullptr;
    }, json_requests);
}

lb_status lb_exports_get(const lb_exports* e, size_t i, const uint8_t** bytes, size_t* len) {
    if (!e || !bytes || !len || i >= e->answers.size()) { g_last_error = "bad argument"; return LB_ERR_INVALID_ARG; }
    const lb_exports::Answer& a = e->answers[i];
    if (a.status != LB_OK) { g_last_error = a.error; return a.status; }
    *bytes = a.bytes;
    *len = a.len;
    return LB_OK;
}

void lb_exports_free(lb_exports* e) { delete e; }

lb_status lb_batch_counters(const lb_batch* b, lb_counters* out) {
    if (!b || !out) return LB_ERR_INVALID_ARG;
    *out = b->counters;
    return LB_OK;
}
lb_status lb_batch_timings(const lb_batch* b, lb_timings* out) {
    if (!b || !out) return LB_ERR_INVALID_ARG;
    *out = b->timings;
    out->alloc_host_ms = (float)b->dev.alloc_ms;
    out->device_bytes = b->dev.bytes;
    return LB_OK;
}

lb_status lb_debug_table(const lb_batch* b, const char* name, void* dst, size_t dst_bytes, size_t* n_elems,
                         size_t* elem_size) {
    if (!b || !name || !n_elems || !elem_size) return LB_ERR_INVALID_ARG;
    if (!(b->flags & LB_FLAG_KEEP_DEVICE)) { g_last_error = "needs LB_FLAG_KEEP_DEVICE"; return LB_ERR_INVALID_ARG; }
    std::string nm(name);
    const void* src = nullptr;
    size_t n = 0, es = 0;
    const BatchTables& t = b->tb;
#define TAB(str, ptr, cnt) if (nm == str) { src = ptr; n = cnt; es = sizeof(*ptr); }
    TAB("op_cid", t.op_cid, b->n.rows) TAB("op_prop", t.op_prop, b->n.rows) TAB("op_vtype", t.op_vtype, b->n.rows)
    TAB("op_len", t.op_len, b->n.rows) TAB("op_counter", t.op_counter, b->n.rows)
    TAB("ch_counter", t.ch_counter, b->n.changes) TAB("ch_len", t.ch_len, b->n.changes)
    TAB("ch_lamport", t.ch_lamport_wire, b->n.changes) TAB("ch_ts", t.ch_ts, b->n.changes)
    TAB("dep_peer", t.dep_peer_idx, b->n.deps) TAB("dep_counter", t.dep_counter, b->n.deps)
#undef TAB
    if (nm == "blk_doc" || nm == "blk_nchanges") {   // fields of the block descriptors
        *n_elems = b->n.blocks;
        *elem_size = 4;
        if (dst) {
            if (dst_bytes < b->n.blocks * 4) { g_last_error = "buffer too small"; return LB_ERR_INVALID_ARG; }
            std::vector<BlockInfo> hb(b->n.blocks);
            if (b->n.blocks && cudaMemcpy(hb.data(), b->tb.blocks, sizeof(BlockInfo) * b->n.blocks, cudaMemcpyDeviceToHost) != cudaSuccess) return LB_ERR_CUDA;
            for (size_t i = 0; i < hb.size(); i++) ((u32*)dst)[i] = nm == "blk_doc" ? hb[i].doc : hb[i].n_changes;
        }
        return LB_OK;
    }
    if (!src) { g_last_error = "unknown table"; return LB_ERR_INVALID_ARG; }
    *n_elems = n;
    *elem_size = es;
    if (dst) {
        if (dst_bytes < n * es) { g_last_error = "buffer too small"; return LB_ERR_INVALID_ARG; }
        if (n && cudaMemcpy(dst, src, n * es, cudaMemcpyDeviceToHost) != cudaSuccess) return LB_ERR_CUDA;
    }
    return LB_OK;
}

void lb_batch_free(lb_batch* b) {
    if (!b) return;
    if (b->json_thread.joinable()) b->json_thread.join();
    if (b->json_ev) cudaEventDestroy(b->json_ev);
    if (b->stream2) cudaStreamDestroy(b->stream2);
    if (b->ev_created) cudaStreamSynchronize(b->dev.stream);   // the cached blocks must be idle
    b->dev.free_all();
    if (b->ev_created) {   // the stream exists whenever the events do (init_batch)
        cudaStreamSynchronize(b->dev.stream);
        for (cudaEvent_t e : b->ev) cudaEventDestroy(e);
        stream_give(b->dev.device, b->dev.stream);
    }
    for (HostResult* r : {&b->json, &b->attr, &b->exported}) lbstage::host_cache().give(r->host);
    delete b;
}

// Give the device blocks kept for the next batch (BlockCache) back to the driver.
lb_status lb_device_trim(int device) {
    lb_options o;
    memset(&o, 0, sizeof(o));
    o.device = device;
    lb_status st = check_device(&o);
    if (st != LB_OK) return st;
    cache_flush(device, nullptr);
    cudaStreamSynchronize(nullptr);
    return LB_OK;
}

// Pin the CALLING thread (and every thread it creates afterwards: the staging workers, the JSON download thread) to
// the CPUs of the NUMA node the device hangs off, so that the pinned staging ring and the gather threads of a rank stay
// next to its GPU.  One process per GPU calls this once, before it builds its input buffers.  LB_ERR_UNSUPPORTED when
// the topology cannot be read (no sysfs entry, single node): nothing is changed.
lb_status lb_numa_bind(int device) {
#ifdef LB_SIMT_EMU
    (void)device;
    g_last_error = "no topology in the emulated build";
    return LB_ERR_UNSUPPORTED;
#else
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { g_last_error = "cudaDeviceGetPCIBusId failed"; return LB_ERR_CUDA; }
    for (char* c = bus; *c; c++) if (*c >= 'A' && *c <= 'Z') *c = (char)(*c - 'A' + 'a');
    std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
    FILE* f = fopen(path.c_str(), "r");
    int node = -1;
    if (f) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
    if (node < 0) { g_last_error = "no NUMA node recorded for " + std::string(bus); return LB_ERR_UNSUPPORTED; }
    path = "/sys/devices/system/node/node" + std::to_string(node) + "/cpulist";
    f = fopen(path.c_str(), "r");
    if (!f) { g_last_error = "cannot read " + path; return LB_ERR_UNSUPPORTED; }
    char list[1024] = {0};
    if (!fgets(list, sizeof(list), f)) list[0] = 0;
    fclose(f);
    cpu_set_t want, have;
    CPU_ZERO(&want);
    for (char* p = list; *p;) {   // "0-31,64-95"
        char* e;
        long a = strtol(p, &e, 10), b_ = a;
        if (e == p) break;
        if (*e == '-') { p = e + 1; b_ = strtol(p, &e, 10); }
        for (long c = a; c <= b_ && c < CPU_SETSIZE; c++) CPU_SET((int)c, &want);
        p = *e == ',' ? e + 1 : e;
        if (*e != ',' ) break;
    }
    if (sched_getaffinity(0, sizeof(have), &have) == 0) {   // stay inside what the container allows
        cpu_set_t both;
        CPU_AND(&both, &want, &have);
        if (CPU_COUNT(&both) == 0) { g_last_error = "the device's NUMA node has no CPU this process may use"; return LB_ERR_UNSUPPORTED; }
        want = both;
    }
    if (sched_setaffinity(0, sizeof(want), &want) != 0) { g_last_error = "sched_setaffinity failed"; return LB_ERR_UNSUPPORTED; }
    return LB_OK;
#endif
}

#ifdef LB_SIMT_EMU
// test hook of the emulated build only: the device-side f64 formatter on the host (tests/test_f64_format.py)
int lb_emu_format_f64(double d, char* out) {
    u64 bits;
    memcpy(&bits, &d, 8);
    return f64_format(bits, out);
}
#endif
}  // extern "C"
