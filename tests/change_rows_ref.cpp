// TEST INFRASTRUCTURE: FastUpdates blobs whose changes hold their ops in pieces.  The oracle document's stored blocks
// are encoded as its all_updates export encodes them, except that every List / Text insert and every delete span is
// first cut (the oracle's Op::slice) into pieces of `piece` atoms, each piece its own op row.  A valid encoding of
// the same changes (the reference writes unmerged neighbours whenever its arenas did not line up), which an importing
// document merges back op by op (block_encode.rs:651): rows of one change that only merge on import, so that the
// export's RleVec merge inside a change (runs across 32-row chunks, single-element deletes merging into directed
// spans, text runs broken by a string-arena doubling of the importer) is exercised.  It lives beside its tests, as
// tests/range_export_ref.cpp does, on the unchanged oracle.  Built by tests/test_export_change_rows_emu.py into a
// temporary directory.
#include "../oracle/doc.hpp"

#include <cstdlib>
#include <cstring>

using namespace lo;

extern "C" {

// Returns 0 and the blob, or -1 and the reason (both malloc'ed).
int cr_export_pieces(void* dp, int piece, uint8_t** out, size_t* len) {
    Doc& d = *(Doc*)dp;
    std::vector<uint8_t> blob;
    std::string err;
    try {
        if (piece < 1) throw std::runtime_error("piece < 1");
        d.commit();
        Writer body;
        for (auto& kv : d.store) {
            std::vector<Change> block;
            for (const Change& c : kv.second.changes) {
                Change r = c;
                r.ops.clear();
                for (const Op& op : c.ops) {
                    const bool cut = op.kind == OP_LIST_INSERT || op.kind == OP_TEXT_INSERT || op.kind == OP_DELETE;
                    const int n = op.atom_len();
                    if (!cut || n <= piece) { r.ops.push_back(op); continue; }
                    for (int a = 0; a < n; a += piece) r.ops.push_back(op_slice(op, a, std::min(n, a + piece)));
                }
                block.push_back(std::move(r));
            }
            std::vector<uint8_t> b = encode_block(block, d);
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

void cr_free(void* p) { std::free(p); }

}  // extern "C"
