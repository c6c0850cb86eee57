// TEST INFRASTRUCTURE: the reference's ExportMode::UpdatesInRange (encoding.rs:52-151, change_store.rs:179-199
// export_blocks_in_range) on top of the oracle, which it reuses unchanged: every span is normalised (span.rs:51-68), the
// oracle document's stored changes that overlap it are cut with the oracle's Change::slice and inserted, in request
// order, into one fresh store with the oracle's insert_change (the previous block by id, merge interval 0), and the store
// is encoded as all_updates is.  Where the reference panics ("counter should be continuous") or would store a change
// twice (spans of one peer that overlap), the call answers an error instead.  It lives beside its tests, as
// tests/json_updates_ref.cpp does, so that the oracle stays the fixed yardstick the other checks are built on.  Built by
// tests/range_export_checks.py into a temporary directory.
#include "../oracle/doc.hpp"

#include <cstdlib>
#include <cstring>

using namespace lo;

extern "C" {

// spans: n entries (peers[i], starts[i], ends[i]).  Returns 0 and the blob, or -1 and the reason (both malloc'ed).
int rx_export(void* dp, const uint64_t* peers, const int32_t* starts, const int32_t* ends, size_t n, uint8_t** out,
              size_t* len) {
    Doc& d = *(Doc*)dp;
    std::vector<uint8_t> blob;
    std::string err;
    try {
        d.commit();
        std::map<ID, StoreBlock> ns;
        std::map<PeerID, std::vector<std::pair<Counter, Counter>>> taken;   // pieces inserted so far, per peer
        for (size_t i = 0; i < n; i++) {
            const PeerID p = peers[i];
            int64_t s = starts[i], e = ends[i];
            if (e < s) { const int64_t s2 = e + 1; e = s + 1; s = s2; }   // CounterSpan::normalize_
            if (s == e) continue;                                       // iter_blocks: empty span
            // iter_blocks starts at the block at or before (peer, start); one of another peer selects nothing
            auto it = d.store.upper_bound(ID{p, (Counter)std::max<int64_t>(s, INT32_MIN)});
            if (it == d.store.begin()) continue;
            --it;
            if (it->first.peer != p) continue;
            for (; it != d.store.end() && it->first.peer == p && it->second.c0 < e; ++it) {
                for (auto& c : it->second.changes) {
                    const int cs = (int)std::min<int64_t>(std::max<int64_t>(s - c.id.counter, 0), c.atom_len());
                    const int ce = (int)std::min<int64_t>(std::max<int64_t>(e - c.id.counter, 0), c.atom_len());
                    if (cs == ce) continue;
                    const Counter a = c.id.counter + cs, b = c.id.counter + ce;
                    for (auto& q : taken[p])
                        if (q.first < b && a < q.second) throw std::runtime_error("spans of one peer overlap");
                    taken[p].push_back({a, b});
                    d.store_insert(ns, (cs == 0 && ce == c.atom_len()) ? c : Doc::change_slice(c, cs, ce), false, 0);
                }
            }
        }
        Writer body;
        for (auto& kv : ns) {
            std::vector<uint8_t> b = encode_block(kv.second.changes, d);
            body.uleb(b.size());
            body.bytes(b);
        }
        blob = wrap_blob(MODE_FAST_UPDATES, body.buf);
    } catch (std::exception& ex) {
        err = ex.what();
    }
    const bool ok = err.empty();
    *len = ok ? blob.size() : err.size();
    *out = (uint8_t*)std::malloc(*len + 1);
    std::memcpy(*out, ok ? blob.data() : (const uint8_t*)err.data(), *len);
    return ok ? 0 : -1;
}

void rx_free(void* p) { std::free(p); }

}  // extern "C"
