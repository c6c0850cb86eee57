// TEST INFRASTRUCTURE: the checkout reference (LoroDoc::checkout(&frontiers) + get_deep_value, loro.rs:1353-1433) on top
// of the oracle, which it reuses unchanged: a copy of an oracle document whose change store holds only the atoms of the
// causal closure of F -- every change cut at V[peer] with the oracle's Change::slice / Op::slice -- replayed by the
// oracle's own replay.  Built by tests/checkout_checks.py into a temporary directory.
#include "../oracle/doc.hpp"

#include <cstdlib>
#include <cstring>

using namespace lo;

namespace {
char* dup_out(const std::string& s, size_t* len) {
    char* p = (char*)std::malloc(s.size() + 1);
    std::memcpy(p, s.data(), s.size());
    p[s.size()] = 0;
    if (len) *len = s.size();
    return p;
}
}  // namespace

extern "C" {

// JSON of document `d` (a handle of oracle/liboracle.so) at the Frontiers (peers[i], ctrs[i]); "!FrontiersNotFound" when an
// id is not an atom of the document's DAG (loro.rs:1394-1410: unknown peer, counter at or past the vv, pending change).
char* ck_json_at(void* d, const uint64_t* peers, const int32_t* ctrs, size_t n, size_t* len) {
    try {
        Doc& src = *(Doc*)d;
        src.commit();
        std::map<PeerID, std::vector<const Change*>> per_peer;   // the store is keyed by id: counter order per peer
        for (auto& kv : src.store)
            for (auto& c : kv.second.changes) per_peer[c.id.peer].push_back(&c);
        auto holding = [&](PeerID p, Counter c) -> const Change* {
            auto it = per_peer.find(p);
            if (it == per_peer.end() || c < 0) return nullptr;
            const auto& v = it->second;
            auto up = std::upper_bound(v.begin(), v.end(), c, [](Counter x, const Change* ch) { return x < ch->id.counter; });
            if (up == v.begin()) return nullptr;
            const Change* ch = *(up - 1);
            return c < ch->ctr_end() ? ch : nullptr;
        };
        std::vector<ID> todo;
        for (size_t i = 0; i < n; i++) {
            if (!holding(peers[i], ctrs[i])) return dup_out("!FrontiersNotFound", len);
            todo.push_back(ID{peers[i], ctrs[i]});
        }
        // V = the causal closure of F: covering [V[p], c + 1) of peer p brings in the deps of every change it touches
        std::map<PeerID, Counter> V;
        while (!todo.empty()) {
            ID id = todo.back();
            todo.pop_back();
            Counter old = V.count(id.peer) ? V[id.peer] : 0;
            if (id.counter < old) continue;
            V[id.peer] = id.counter + 1;
            for (const Change* ch : per_peer[id.peer]) {
                if (ch->ctr_end() <= old || ch->id.counter > id.counter) continue;
                for (const ID& dep : ch->deps) todo.push_back(dep);
            }
        }
        Doc cp = src;
        for (auto it = cp.store.begin(); it != cp.store.end();) {
            std::vector<Change> kept;
            for (Change& c : it->second.changes) {
                Counter cap = V.count(c.id.peer) ? V[c.id.peer] : 0;
                if (c.id.counter >= cap) continue;
                if (c.ctr_end() > cap) kept.push_back(Doc::change_slice(c, 0, cap - c.id.counter));
                else kept.push_back(std::move(c));
            }
            it->second.changes = std::move(kept);
            if (it->second.changes.empty()) it = cp.store.erase(it);
            else ++it;
        }
        for (auto& kv : cp.vv) kv.second = V.count(kv.first) ? V[kv.first] : 0;
        cp.pending.clear();
        cp.state_valid = false;
        return dup_out(cp.to_json(), len);
    } catch (std::exception& e) {
        return dup_out(std::string("!error: ") + e.what(), len);
    }
}

void ck_free(void* p) { std::free(p); }
}
