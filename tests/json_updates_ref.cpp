// TEST INFRASTRUCTURE: the JSON-updates reference (LoroDoc::export_json_updates, loro.rs:715-751, encoding/json_schema.rs)
// on top of the oracle, which it reuses unchanged: the oracle document's own change store walked peer by peer, every
// change overlapping [start, end) cut with the oracle's Change::slice, sorted stably by lamport (equal lamports by
// ascending peer id), the peers registered in encode_change's order and the text printed as serde_json prints the `json`
// module.  Built by tests/json_updates_checks.py into a temporary directory.
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

struct JsonWriter {
    Doc& d;
    bool compress;
    std::vector<PeerID> peers;
    std::map<PeerID, size_t> index;
    std::string out;

    PeerID reg(PeerID p) {   // ValueRegister::register (encoding/value_register.rs)
        if (!compress) return p;
        auto it = index.find(p);
        if (it != index.end()) return it->second;
        index[p] = peers.size();
        peers.push_back(p);
        return peers.size() - 1;
    }
    static const char* type_name(uint8_t t) {
        static const char* names[6] = {"Map", "List", "Text", "Tree", "MovableList", "Counter"};
        return t < 6 ? names[t] : "Unknown";
    }
    std::string cid(const ContainerID& c) {   // ContainerID Display, loro-common/src/lib.rs:480-500
        if (c.root) return "cid:root-" + c.name + ":" + type_name(c.type);
        return "cid:" + std::to_string(c.counter) + "@" + std::to_string(reg(c.peer)) + ":" + type_name(c.type);
    }
    std::string id(PeerID p, Counter c) { return "\"" + std::to_string(c) + "@" + std::to_string(reg(p)) + "\""; }
    void value(std::string& o, const Value& v) {   // LoroValue's serde (value.rs:692-711), object keys ascending
        switch (v.k) {
            case Value::List:
                o += "[";
                for (size_t i = 0; i < v.list.size(); i++) { if (i) o += ","; value(o, v.list[i]); }
                o += "]";
                break;
            case Value::Map: {
                std::vector<const std::pair<std::string, Value>*> es;
                for (auto& kv : v.map) es.push_back(&kv);
                std::stable_sort(es.begin(), es.end(), [](auto a, auto b) { return a->first < b->first; });
                o += "{";
                bool first = true;
                for (size_t i = 0; i < es.size(); i++) {
                    if (i + 1 < es.size() && es[i + 1]->first == es[i]->first) continue;   // the later one wins
                    if (!first) o += ",";
                    first = false;
                    json_escape(o, es[i]->first);
                    o += ":";
                    value(o, es[i]->second);
                }
                o += "}";
                break;
            }
            case Value::Container: json_escape(o, "🦜:" + cid(v.cid)); break;
            default: d.json_value(o, v, 0);
        }
    }
    // encode_change (json_schema.rs:301-548): the ops register first, then the change id, then the sorted deps
    void change(const Change& c) {
        std::string ops;
        for (size_t k = 0; k < c.ops.size(); k++) {
            const Op& op = c.ops[k];
            std::string o = "{\"container\":";
            json_escape(o, cid(d.containers[(size_t)op.cidx]));
            o += ",\"content\":{\"type\":";
            switch (op.kind) {
                case OP_LIST_INSERT: {
                    o += "\"insert\",\"pos\":" + std::to_string(op.prop) + ",\"value\":[";
                    for (size_t i = 0; i < op.values.size(); i++) { if (i) o += ","; value(o, op.values[i]); }
                    o += "]";
                    break;
                }
                case OP_TEXT_INSERT:
                    o += "\"insert\",\"pos\":" + std::to_string(op.prop) + ",\"text\":";
                    json_escape(o, op.text);
                    break;
                case OP_DELETE:
                    o += "\"delete\",\"pos\":" + std::to_string(op.prop) + ",\"len\":" + std::to_string(op.del_len) +
                         ",\"start_id\":" + id(op.del_start.peer, op.del_start.counter);
                    break;
                case OP_MAP_SET: case OP_MAP_DEL:
                    o += op.kind == OP_MAP_SET ? "\"insert\",\"key\":" : "\"delete\",\"key\":";
                    json_escape(o, op.key);
                    if (op.kind == OP_MAP_SET) { o += ",\"value\":"; value(o, op.mapval); }
                    break;
                case OP_TREE_CREATE: case OP_TREE_MOVE: case OP_TREE_DELETE: {
                    o += op.kind == OP_TREE_CREATE ? "\"create\"" : op.kind == OP_TREE_MOVE ? "\"move\"" : "\"delete\"";
                    o += ",\"target\":" + id(op.target.peer, op.target.counter);
                    if (op.kind != OP_TREE_DELETE) {
                        o += ",\"parent\":" + (op.parent_null ? std::string("null") : id(op.parent.peer, op.parent.counter));
                        o += ",\"fractional_index\":\"";
                        static const char* HEX = "0123456789ABCDEF";
                        for (unsigned char b : op.position) { o.push_back(HEX[b >> 4]); o.push_back(HEX[b & 15]); }
                        o += "\"";
                    }
                    break;
                }
                default: throw std::runtime_error("op kind outside the JSON export");
            }
            o += "},\"counter\":" + std::to_string(op.counter) + "}";
            if (k) ops += ",";
            ops += o;
        }
        std::string head = "{\"id\":" + id(c.id.peer, c.id.counter) + ",\"timestamp\":" + std::to_string(c.timestamp) +
                           ",\"deps\":[";
        std::vector<ID> deps = c.deps;
        std::sort(deps.begin(), deps.end());
        for (size_t k = 0; k < deps.size(); k++) { if (k) head += ","; head += id(deps[k].peer, deps[k].counter); }
        head += "],\"lamport\":" + std::to_string(c.lamport) + ",\"msg\":";
        if (c.has_msg) json_escape(head, c.msg); else head += "null";
        out += head + ",\"ops\":[" + ops + "]}";
    }
};

std::map<PeerID, Counter> refine(const Doc& d, const uint64_t* peers, const int32_t* ctrs, size_t n) {   // json_schema.rs:31-45
    std::map<PeerID, Counter> r;
    for (size_t i = 0; i < n; i++) {
        if (ctrs[i] == 0) { r.erase(peers[i]); continue; }
        auto it = d.vv.find(peers[i]);
        Counter end = it == d.vv.end() ? 0 : it->second;
        r[peers[i]] = std::max(0, std::min(end, ctrs[i]));
    }
    return r;
}
}  // namespace

extern "C" {

// export_json_updates(start, end, peer_compression) of oracle document `d` as serde_json text
char* jx_export(void* dp, const uint64_t* sp, const int32_t* sc, size_t ns, const uint64_t* ep, const int32_t* ec, size_t ne,
                int compress, size_t* len) {
    try {
        Doc& d = *(Doc*)dp;
        d.commit();
        std::map<PeerID, Counter> S = refine(d, sp, sc, ns), E = refine(d, ep, ec, ne);
        std::map<PeerID, std::vector<const Change*>> per_peer;   // the store is keyed by id: counter order per peer
        for (auto& kv : d.store)
            for (auto& c : kv.second.changes) per_peer[c.id.peer].push_back(&c);
        std::vector<Change> picked;
        for (auto& kv : per_peer) {   // iter_changes_peer_by_peer + init_encode (json_schema.rs:144-169)
            Counter s = S.count(kv.first) ? S[kv.first] : 0, e = E.count(kv.first) ? E[kv.first] : 0;
            if (s >= e) continue;
            for (const Change* c : kv.second) {
                if (c->ctr_end() <= s || c->id.counter >= e) continue;
                int from = std::max(0, s - c->id.counter), to = std::min(c->atom_len(), e - c->id.counter);
                picked.push_back(from == 0 && to == c->atom_len() ? *c : Doc::change_slice(*c, from, to));
            }
        }
        std::stable_sort(picked.begin(), picked.end(), [](const Change& a, const Change& b) { return a.lamport < b.lamport; });
        // vv_to_frontiers (loro_dag.rs:1036-1065): the last ids of the start, without those in another one's causal past
        std::map<ID, std::map<PeerID, Counter>> past;   // id -> vv of its causal past, including itself
        std::function<std::map<PeerID, Counter>(ID)> vv_of = [&](ID id) -> std::map<PeerID, Counter> {
            auto it = past.find(id);
            if (it != past.end()) return it->second;
            std::map<PeerID, Counter> v;
            std::vector<ID> todo{id};
            while (!todo.empty()) {
                ID x = todo.back();
                todo.pop_back();
                if (v.count(x.peer) && v[x.peer] > x.counter) continue;
                Counter old = v.count(x.peer) ? v[x.peer] : 0;
                v[x.peer] = x.counter + 1;
                for (const Change* c : per_peer[x.peer]) {
                    if (c->ctr_end() <= old || c->id.counter > x.counter) continue;
                    for (const ID& dep : c->deps) todo.push_back(dep);
                }
            }
            return past[id] = v;
        };
        JsonWriter w{d, compress != 0, {}, {}, {}};
        std::string body;
        for (const Change& c : picked) {
            w.out.clear();
            w.change(c);
            if (!body.empty()) body += ",";
            body += w.out;
        }
        std::string o = "{\"schema_version\":1,\"start_version\":{";
        bool first = true;
        for (auto& kv : S) {
            if (kv.second <= 0) continue;
            bool covered = false;
            for (auto& q : S)
                if (q.first != kv.first && q.second > 0) {
                    auto v = vv_of(ID{q.first, q.second - 1});
                    if (v.count(kv.first) && v[kv.first] >= kv.second) covered = true;
                }
            if (covered) continue;
            if (!first) o += ",";
            first = false;
            o += "\"" + std::to_string(kv.first) + "\":" + std::to_string(kv.second - 1);
        }
        o += "},\"peers\":";
        if (compress) {
            o += "[";
            for (size_t i = 0; i < w.peers.size(); i++) { if (i) o += ","; o += "\"" + std::to_string(w.peers[i]) + "\""; }
            o += "]";
        } else o += "null";
        o += ",\"changes\":[" + body + "]}";
        return dup_out(o, len);
    } catch (std::exception& e) {
        return dup_out(std::string("!error: ") + e.what(), len);
    }
}

// commit the open transaction with a timestamp and a message (the oracle's own commit records neither)
void jx_commit_with(void* dp, int64_t timestamp, const char* msg, size_t msg_len, int has_msg) {
    Doc& d = *(Doc*)dp;
    if (d.txn_open) {
        d.txn.timestamp = timestamp;
        d.txn.has_msg = has_msg != 0;
        d.txn.msg.assign(msg ? msg : "", msg ? msg_len : 0);
    }
    d.commit();
}

void jx_free(void* p) { std::free(p); }
}
