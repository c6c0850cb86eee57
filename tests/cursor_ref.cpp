// TEST INFRASTRUCTURE: LoroDoc::get_cursor_pos (crates/loro-internal/src/loro.rs:1560-1737 query_pos_internal) restated on
// the oracle, which it reuses unchanged.  Two sources, as in the reference:
//   * a visible target is looked up in the oracle's materialised state (`ids` of the Text / List: state.rs:1403-1433);
//   * a deleted one needs a delete op of the container that covers it (find_last_delete_op, loro.rs:2003-2022), then
//     its position among the spans of the tracker's rope (tracker.rs:588-619).  The oracle's replay drops its trackers,
//     so this file replays the document's Text / List ops once more with the oracle's Tracker, in the oracle's order,
//     and keeps the ropes.
// The update cursor is get_cursor(pos, side) on the state (handler.rs:2337-2390, :2912-2952).  Built by
// tests/cursor_checks.py into a temporary directory.
#include "../oracle/doc.hpp"

#include <cstdlib>
#include <map>
#include <memory>
#include <set>

using namespace lo;

namespace {
struct RopeSpan {
    PeerID peer;
    Counter ctr;
    int len;
    bool active;
};
struct Ctx {
    Doc* doc;
    std::map<int, std::vector<RopeSpan>> ropes;   // container index -> every span of its final rope, in order
};

// the Text / List part of Doc::replay (oracle/doc.hpp), keeping each container's tracker rope at the end
void replay_ropes(Doc& doc, Ctx& cx) {
    std::vector<PeerID> peer_ids;
    std::map<PeerID, int> pidx;
    for (auto& kv : doc.vv) {
        pidx[kv.first] = (int)peer_ids.size();
        peer_ids.push_back(kv.first);
    }
    const int P = (int)peer_ids.size();
    std::vector<std::vector<const Change*>> per_peer((size_t)P);
    for (auto& kv : doc.store)
        for (auto& c : kv.second.changes) per_peer[(size_t)pidx[c.id.peer]].push_back(&c);
    std::vector<std::vector<std::vector<Counter>>> cvv((size_t)P);
    for (int p = 0; p < P; p++) cvv[(size_t)p].resize(per_peer[(size_t)p].size());
    auto find_idx = [&](int p, Counter c) -> int {
        auto& v = per_peer[(size_t)p];
        int lo = 0, hi = (int)v.size() - 1, ans = -1;
        while (lo <= hi) {
            int mid = (lo + hi) / 2;
            if (v[(size_t)mid]->id.counter <= c) { ans = mid; lo = mid + 1; } else hi = mid - 1;
        }
        return ans;
    };
    std::vector<size_t> next((size_t)P, 0);
    std::vector<Counter> applied((size_t)P, 0);
    auto ready = [&](const Change* c) {
        for (auto& d : c->deps) {
            auto it = pidx.find(d.peer);
            if (it == pidx.end() || applied[(size_t)it->second] <= d.counter) return false;
        }
        return true;
    };
    std::map<int, std::unique_ptr<Tracker>> trackers;
    size_t total = 0;
    for (auto& v : per_peer) total += v.size();
    int cur_peer = -1;
    for (size_t done = 0; done < total; done++) {
        int pick = -1;
        if (cur_peer >= 0 && next[(size_t)cur_peer] < per_peer[(size_t)cur_peer].size() &&
            ready(per_peer[(size_t)cur_peer][next[(size_t)cur_peer]]))
            pick = cur_peer;
        else {
            Lamport best = 0;
            for (int p = 0; p < P; p++) {
                if (next[(size_t)p] >= per_peer[(size_t)p].size()) continue;
                const Change* c = per_peer[(size_t)p][next[(size_t)p]];
                if (!ready(c)) continue;
                if (pick < 0 || c->lamport < best) { pick = p; best = c->lamport; }
            }
        }
        if (pick < 0) throw std::runtime_error("replay: no ready change");
        cur_peer = pick;
        size_t ci = next[(size_t)pick]++;
        const Change* c = per_peer[(size_t)pick][ci];
        std::vector<Counter> v((size_t)P, 0);
        for (auto& d : c->deps) {
            int dp = pidx[d.peer];
            const std::vector<Counter>& dv = cvv[(size_t)dp][(size_t)find_idx(dp, d.counter)];
            for (int q = 0; q < P; q++) v[(size_t)q] = std::max(v[(size_t)q], dv[(size_t)q]);
            v[(size_t)dp] = std::max(v[(size_t)dp], d.counter + 1);
        }
        cvv[(size_t)pick][ci] = v;
        std::set<int> visited;
        for (const Op& op : c->ops) {
            if (op.kind != OP_LIST_INSERT && op.kind != OP_TEXT_INSERT && op.kind != OP_DELETE) continue;
            auto& tp = trackers[op.cidx];
            if (!tp) tp.reset(new Tracker(P));
            Tracker& t = *tp;
            if (visited.insert(op.cidx).second) {
                std::vector<Counter> ov = v;
                ov[(size_t)pick] = std::max(ov[(size_t)pick], op.counter);
                t.checkout(ov);
            }
            if (op.kind == OP_DELETE) {
                auto f = pidx.find(op.del_start.peer);
                t.del(pick, op.counter, f == pidx.end() ? -2 : f->second, op.del_start.counter, op.del_start_pos(),
                      op.atom_len(), op.del_len < 0);
            } else {
                t.insert(pick, op.counter, op.atom_len(), op.prop, peer_ids[(size_t)pick], peer_ids);
            }
        }
        applied[(size_t)pick] = c->ctr_end();
    }
    for (auto& kv : trackers) {
        Tracker& t = *kv.second;
        t.checkout(applied);
        std::vector<RopeSpan>& rope = cx.ropes[kv.first];
        for (auto& blk : t.blocks)
            for (TSpan* s : blk.spans)
                if (s->peer >= 0) rope.push_back(RopeSpan{peer_ids[(size_t)s->peer], s->ctr, s->len, s->active()});
    }
}
}  // namespace

extern "C" {

// a query context on document `d` (a handle of oracle/liboracle.so), valid while the document is not changed
void* cr_open(void* d) {
    try {
        Doc& doc = *(Doc*)d;
        doc.commit();
        doc.ensure_state();
        Ctx* cx = new Ctx();
        cx->doc = &doc;
        replay_ropes(doc, *cx);
        return cx;
    } catch (std::exception&) {
        return nullptr;
    }
}

void cr_close(void* p) { delete (Ctx*)p; }

// out: status (0, 100 IdNotFound, 1 the container type has no answer), pos, side, has_update, update_has_id,
// update_peer, update_counter, update_side, update_origin_pos
void cr_query(void* p, int is_root, const char* name, size_t name_len, uint64_t cpeer, int32_t ccounter, int type, int has_id,
              uint64_t id_peer, int32_t id_counter, int side, int64_t* out) {
    Ctx& cx = *(Ctx*)p;
    Doc& doc = *cx.doc;
    for (int k = 0; k < 9; k++) out[k] = 0;
    out[2] = side;
    if (type != CT_TEXT && type != CT_LIST) { out[0] = 1; return; }   // unreachable!() in the reference
    ContainerID cid;
    cid.root = is_root != 0;
    cid.type = (uint8_t)type;
    if (cid.root) cid.name.assign(name, name_len);
    else { cid.peer = cpeer; cid.counter = ccounter; }
    auto it = doc.cid_index.find(cid);
    // has_container (loro.rs:889-896): a root always exists, a normal container when the document registered it
    if (it == doc.cid_index.end() && !cid.root) { out[0] = 100; return; }
    const int cidx = it == doc.cid_index.end() ? -1 : it->second;
    static const std::vector<ID> none;
    const std::vector<ID>& ids = cidx >= 0 && (size_t)cidx < doc.state.size() ? doc.state[(size_t)cidx].ids : none;
    const int64_t len = (int64_t)ids.size();
    if (!has_id) { out[1] = side == -1 ? 0 : len; return; }
    const ID id{id_peer, id_counter};
    for (size_t k = 0; k < ids.size(); k++)
        if (ids[k] == id) { out[1] = (int64_t)k; return; }
    // find_last_delete_op: a delete op of this container whose target span holds the id
    bool deleted = false;
    for (auto& kv : doc.store)
        for (const Change& c : kv.second.changes)
            for (const Op& op : c.ops)
                if (op.cidx == cidx && op.kind == OP_DELETE && op.del_start.peer == id.peer &&
                    id.counter >= op.del_start.counter && id.counter < op.del_start.counter + op.atom_len())
                    deleted = true;
    if (!deleted) { out[0] = 100; return; }
    // get_target_id_latest_index_at_new_version (tracker.rs:588-619)
    int64_t pos = 0;
    bool found = false, active = false;
    for (const RopeSpan& s : cx.ropes[cidx]) {
        if (s.peer == id.peer && id.counter >= s.ctr && id.counter < s.ctr + s.len) {
            if (s.active) pos += id.counter - s.ctr;
            found = true;
            active = s.active;
            break;
        }
        if (s.active) pos += s.len;
    }
    if (!found) { out[0] = 100; return; }
    const int rside = active ? 0 : -1;
    out[1] = pos;
    out[2] = rside;
    out[3] = 1;
    if (len == 0) { out[7] = rside == 0 ? -1 : rside; out[8] = 0; }
    else if (pos >= len) { out[7] = 1; out[8] = len; }
    else {
        out[4] = 1;
        out[5] = (int64_t)ids[(size_t)pos].peer;
        out[6] = ids[(size_t)pos].counter;
        out[7] = rside;
        out[8] = pos;
    }
}
}
