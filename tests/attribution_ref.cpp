// TEST INFRASTRUCTURE: the attribution reference on top of the oracle, which it reuses unchanged.  The sources are the
// oracle's materialised ContainerState after its own replay: `ids` of a Text / List (LoroText::get_editor_at_unicode_pos,
// LoroList::get_id_at), the MapEntry of every key (lamport and peer of the winning op, deletes included:
// LoroMap::get_last_editor), the TreeNodeState of every node (lamport and peer of its last effective move, whose counter
// is recovered through the change store: LoroTree::get_last_move_id).  At Frontiers F the document is the checkout
// reference's capped copy (tests/checkout_ref.cpp): every change cut at the causal closure of F with the oracle's
// Change::slice.  Printed in the engine's canonical form (include/loro_b200.h lb_doc_attribution).  Built by
// tests/attribution_checks.py into a temporary directory.
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

const char* type_name(uint8_t t) {
    static const char* names[6] = {"Map", "List", "Text", "Tree", "MovableList", "Counter"};
    return t < 6 ? names[t] : "Unknown";
}

// `cp` (a copy of `src`) cut to the atoms of the causal closure of `f` (false: an id of f is not in the DAG)
bool capped_copy(Doc& src, const std::vector<ID>& f, Doc& cp) {
    std::map<PeerID, std::vector<const Change*>> per_peer;
    for (auto& kv : src.store)
        for (auto& c : kv.second.changes) per_peer[c.id.peer].push_back(&c);
    auto holding = [&](PeerID p, Counter c) -> bool {
        auto it = per_peer.find(p);
        if (it == per_peer.end() || c < 0) return false;
        for (const Change* ch : it->second)
            if (c >= ch->id.counter && c < ch->ctr_end()) return true;
        return false;
    };
    std::vector<ID> todo;
    for (const ID& id : f) {
        if (!holding(id.peer, id.counter)) return false;
        todo.push_back(id);
    }
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
    return true;
}
}  // namespace

extern "C" {

// attribution of document `d` (a handle of oracle/liboracle.so): at Frontiers (peers[i], ctrs[i]) when `at`, else at the
// latest version; "!FrontiersNotFound" when an id of F is not an atom of the document's DAG
char* at_attribution(void* d, int at, const uint64_t* peers, const int32_t* ctrs, size_t n, size_t* len) {
    try {
        Doc& src = *(Doc*)d;
        src.commit();
        Doc cp = src;
        if (at) {
            std::vector<ID> f;
            for (size_t i = 0; i < n; i++) f.push_back(ID{peers[i], ctrs[i]});
            if (!capped_copy(src, f, cp)) return dup_out("!FrontiersNotFound", len);
        }
        cp.state_valid = false;   // the replayed state, also for a document edited locally
        cp.ensure_state();
        // peers of the oplog vv, ascending
        std::map<PeerID, size_t> vix;
        std::string out = "{\"peers\":[";
        for (auto& kv : src.vv) {
            if (kv.second <= 0) continue;
            if (!vix.empty()) out.push_back(',');
            out += "\"" + std::to_string(kv.first) + "\"";
            vix.emplace(kv.first, vix.size());
        }
        out += "],\"containers\":{";
        // the counter of peer p's op at lamport l (tree moves are one atom each)
        auto counter_at = [&](PeerID p, Lamport l) -> Counter {
            for (auto& kv : cp.store)
                for (const Change& c : kv.second.changes)
                    if (c.id.peer == p && l >= c.lamport && l < c.lamport_end()) return c.id.counter + (Counter)(l - c.lamport);
            throw std::runtime_error("tree move not in the change store");
        };
        std::vector<size_t> order;
        for (size_t i = 0; i < cp.containers.size(); i++) order.push_back(i);
        std::sort(order.begin(), order.end(), [&](size_t a, size_t b) {
            const ContainerID& x = cp.containers[a];
            const ContainerID& y = cp.containers[b];
            if (x.root != y.root) return x.root;
            if (x.root) return x.name != y.name ? x.name < y.name : x.type < y.type;
            if (x.peer != y.peer) return x.peer < y.peer;
            return x.counter != y.counter ? x.counter < y.counter : x.type < y.type;
        });
        bool first = true;
        for (size_t i : order) {
            if (i >= cp.state.size()) continue;
            const ContainerID& cid = cp.containers[i];
            const ContainerState& st = cp.state[i];
            std::string entry;
            if (cid.type == CT_TEXT || cid.type == CT_LIST) {
                if (st.ids.empty()) continue;
                entry = "[";
                for (size_t k = 0; k < st.ids.size();) {
                    size_t e = k + 1;
                    while (e < st.ids.size() && st.ids[e].peer == st.ids[k].peer &&
                           st.ids[e].counter == st.ids[k].counter + (Counter)(e - k)) e++;
                    if (k) entry.push_back(',');
                    entry += "[" + std::to_string(vix.at(st.ids[k].peer)) + "," + std::to_string(st.ids[k].counter) + "," +
                             std::to_string(e - k) + "]";
                    k = e;
                }
                entry += "]";
            } else if (cid.type == CT_MAP) {
                bool any = false;
                entry = "{";
                for (auto& kv : st.map) {
                    if (!kv.second.set) continue;
                    if (any) entry.push_back(',');
                    any = true;
                    json_escape(entry, kv.first);
                    entry += ":[" + std::to_string(vix.at(kv.second.peer)) + "," + std::to_string(kv.second.lamport) + "," +
                             (kv.second.has ? "1" : "0") + "]";
                }
                entry += "}";
                if (!any) continue;
            } else if (cid.type == CT_TREE) {
                if (st.tree.empty()) continue;
                std::vector<const TreeNodeState*> nodes;
                for (auto& nd : st.tree) nodes.push_back(&nd);
                std::sort(nodes.begin(), nodes.end(), [](const TreeNodeState* a, const TreeNodeState* b) {
                    return a->id.peer != b->id.peer ? a->id.peer < b->id.peer : a->id.counter < b->id.counter;
                });
                entry = "{";
                for (size_t k = 0; k < nodes.size(); k++) {
                    const TreeNodeState* nd = nodes[k];
                    if (k) entry.push_back(',');
                    entry += "\"" + id_string(nd->id) + "\":[" + std::to_string(vix.at(nd->peer)) + "," +
                             std::to_string(counter_at(nd->peer, nd->lamport)) + "," + (nd->deleted ? "0" : "1") + "]";
                }
                entry += "}";
            } else {
                continue;
            }
            if (!first) out.push_back(',');
            first = false;
            std::string name = cid.root ? "cid:root-" + cid.name
                                        : "cid:" + std::to_string(cid.counter) + "@" + std::to_string(cid.peer);
            json_escape(out, name + ":" + type_name(cid.type));
            out.push_back(':');
            out += entry;
        }
        out += "}}";
        return dup_out(out, len);
    } catch (std::exception& e) {
        return dup_out(std::string("!error: ") + e.what(), len);
    }
}

void at_free(void* p) { std::free(p); }
}
