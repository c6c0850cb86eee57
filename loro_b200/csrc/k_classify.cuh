// loro_b200 -- phase 4: per-op-row classification, atom->row index, map last-writer-wins.
//
// Replaces (reference, relative to crates/loro-internal/src):
//   encoding/outdated_encode_reordered.rs:215-423 decode_op (value kind x container type -> op content)
//   diff_calc.rs:423-551 MapDiffCalculator + delta/map_delta.rs:19-46 (LWW by (lamport, peer))
// Fully data-parallel: one thread per op row; the LWW reduce is an atomicMax over a packed
// (lamport, peer rank) key followed by a pass that elects the matching row.
#pragma once
#include "lb_tables.cuh"

__device__ __forceinline__ u8 classify_op(u8 ctype, u8 vt) {
    switch (ctype) {
        case CT_TEXT:
            if (vt == VK_STR) return OPK_SEQ_INS;
            if (vt == VK_DELETE_SEQ) return OPK_SEQ_DEL;
            return OPK_UNSUPPORTED;  // MarkStart / Null (style anchors): SURVEY 8f.2
        case CT_LIST:
            if (vt == VK_LORO_VALUE) return OPK_SEQ_INS;
            if (vt == VK_DELETE_SEQ) return OPK_SEQ_DEL;
            return OPK_UNSUPPORTED;
        case CT_MAP:
            if (vt == VK_LORO_VALUE) return OPK_MAP_SET;
            if (vt == VK_DELETE_ONCE) return OPK_MAP_DEL;
            return OPK_UNSUPPORTED;
        case CT_TREE:
            if (vt == VK_RAW_TREE_MOVE) return OPK_TREE;
            return OPK_UNSUPPORTED;
        default: return OPK_UNSUPPORTED;  // movable list, counter, unknown
    }
}

__global__ void k_op_classify(DocInfo* __restrict__ docs, u64 n_rows, const __grid_constant__ BatchTables t) {
    u64 row = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    u32 ch = t.op_change[row];
    const BlockInfo& bi = t.blocks[t.ch_block[ch]];
    DocInfo& di = docs[bi.doc];
    if (di.code != DOC_OK) {
        t.op_kind[row] = OPK_SKIP;
        uint4 z; z.x = z.y = z.z = z.w = 0;
        t.op_rec[row] = z;
        return;
    }
    u32 cidx = t.cid_map[bi.cid0 + t.op_cid[row]];
    DocContainer& dc = t.dcont[di.cid0 + cidx];
    u8 kind = classify_op(dc.type, t.op_vtype[row]);
    if (kind == OPK_SEQ_INS && dc.type == CT_LIST) {
        // a List insert carries LoroValue::List with exactly `len` items (outdated_encode_reordered.rs:246-262: the
        // reference fails the import otherwise); later phases address the items through `len`
        Cur pk(t.bytes + t.op_val_off[row], t.op_val_len[row]);
        u8 k = pk.get();
        u64 n_items = pk.varint();
        if (pk.err || k != 7 || n_items != (u64)t.op_len[row]) { kind = OPK_SKIP; di.code = LB_ERR(DOC_ERR_CORRUPT); }
    }
    if ((kind == OPK_MAP_SET || kind == OPK_MAP_DEL) && (u32)t.op_prop[row] >= bi.n_keys) {
        kind = OPK_SKIP;                       // a map op whose key index is outside the block's key arena
        di.code = LB_ERR(DOC_ERR_CORRUPT);      // (any thread may write it: every writer stores the same code)
    }
    if (!t.ch_applied[ch]) kind = OPK_SKIP;
    // a change whose head was already known arrives as a slice: rows before the cut are dropped, the row under the cut
    // loses its first `cut_skip` atoms (Op::slice, list_op.rs:603-658)
    u32 cut_skip = 0;
    if (t.ch_trim[ch]) {
        i32 cut = t.ch_counter[ch] + (i32)t.ch_trim[ch];
        if (t.op_counter[row] + (i32)t.op_len[row] <= cut) kind = OPK_SKIP;
        else if (t.op_counter[row] < cut) cut_skip = (u32)(cut - t.op_counter[row]);
    }
    // checkout (k_checkout.cuh): the mirror at the other end -- a row wholly at or past the requested version is no part
    // of the state, the row under the cut loses its last `cut_tail` atoms.  Both cuts can hit one row.
    u32 cut_tail = 0;
    bool beyond = false;
    if (t.ck_end) {
        const i32 end = t.ck_end[di.peer0 + t.ch_peer[ch]];
        const i32 row_end = t.op_counter[row] + (i32)t.op_len[row];
        if (t.op_counter[row] + (i32)cut_skip >= end) beyond = true;
        else if (row_end > end) cut_tail = (u32)(row_end - end);
    }
    u32 lam = t.ch_lamport[ch] + (u32)(t.op_counter[row] - t.ch_counter[ch]);
    if (kind != OPK_TREE && t.op_vtype[row] == VK_RAW_TREE_MOVE) {
        // a RawTreeMove row that is not an applied op of a Tree container: its slot of the tree tables says so (the
        // tree kernel skips it; the tables are not pre-filled)
        u32 ti = t.op_del[row];
        t.tr_rec[ti].w = 0xFFFFFFFFu;
        t.tr_key[ti] = ~0ull;
    }
    if (kind == OPK_TREE) {
        // target and parent must be atoms the document holds: an applied move causally follows the creation of both
        // nodes (tree ids are the ids of the create ops: loro-common/src/lib.rs TreeID)
        u32 ti = t.op_del[row];
        u32 tp = t.peer_map[bi.peer0 + t.tr_target_peer[ti]];
        i32 tc = t.tr_target_ctr[ti];
        u8 pk = t.tr_parent_kind[ti];
        bool ok = tp < di.P && tc >= 0 && tc < t.dpeer[di.peer0 + tp].end_counter;
        u32 pa = pk == TRP_ROOT ? TREE_ROOT : TREE_DELETED;
        u32 pp = pk == TRP_ROOT ? 0u : t.peer_map[bi.peer0 + t.tr_parent_peer[ti]];
        i32 pc = t.tr_parent_ctr[ti];
        if (ok && pk == TRP_NODE) {
            ok = pp < di.P && pc >= 0 && pc < t.dpeer[di.peer0 + pp].end_counter;
            if (ok) pa = t.dpeer[di.peer0 + pp].atom_base + (u32)pc;
        }
        if (!ok) { kind = OPK_SKIP; di.code = LB_ERR(DOC_ERR_CORRUPT); t.tr_rec[ti].w = 0xFFFFFFFFu; t.tr_key[ti] = ~0ull; }
        else {
            uint4 tr;
            tr.x = t.dpeer[di.peer0 + tp].atom_base + (u32)tc;
            tr.y = pa;
            tr.z = t.tr_pos[ti];
            tr.w = (u32)row;
            t.tr_rec[ti] = tr;
            uint4 ids;
            ids.x = tp; ids.y = (u32)tc; ids.z = (u32)pk | (pp << 2); ids.w = (u32)pc;
            t.tr_ids[ti] = ids;
            t.tr_key[ti] = ((u64)lam << 32) | ((u64)t.dpeer[di.peer0 + t.ch_peer[ch]].rank << 16);
            if (beyond) { t.tr_rec[ti].w = 0xFFFFFFFFu; t.tr_key[ti] = ~0ull; }
        }
    }
    {   // tracker record: everything k_seq needs about this row in one 16-byte load
        u32 w = (u32)t.op_prop[row], aux = 0, rev = 0;
        if (kind == OPK_SEQ_DEL) {
            u32 dl = t.op_del[row];
            i32 dlen = t.del_len[dl];
            u32 tp = t.peer_map[bi.peer0 + t.del_peer_idx[dl]];
            i32 tc = t.del_counter[dl];
            i32 n = (i32)t.op_len[row];
            // the target atoms must exist: an applied delete causally follows the inserts it removes
            if (tp >= di.P || tc < 0 || (i64)tc + n > (i64)t.dpeer[di.peer0 + tp].end_counter) kind = OPK_UNSUPPORTED;
            w = (u32)tc;
            aux = tp;
            rev = dlen < 0 ? 1u : 0u;
            if (cut_skip && !rev) w += cut_skip;   // forward span: the first targets go with the dropped atoms
            if (rev) w += cut_tail;                // reversed span: the last atoms delete the lowest targets
                                                   // (DeleteSpanWithId::slice, container/list/list_op.rs:251-270)
        } else if (kind == OPK_SEQ_INS) w += cut_skip;   // insert position of the first kept atom
        if (beyond) {   // unsupported ops are counted over the whole applied history, wherever they fall
            if (kind == OPK_UNSUPPORTED) atomicAdd(&di.has_unsupported, 1u);
            kind = OPK_SKIP;
        }
        uint4 rec;
        rec.x = (u32)kind | (rev << 3) | (cidx << 4);
        rec.y = (u32)t.op_counter[row] + cut_skip;
        rec.z = t.op_len[row] - cut_skip - cut_tail;
        rec.w = w;
        t.op_rec[row] = rec;
        t.op_aux[row] = aux;
    }
    t.op_kind[row] = kind;
    t.op_cidx[row] = cidx;
    t.op_lamport[row] = lam;
    if (kind == OPK_SKIP) return;
    u32 len = t.op_len[row] - cut_skip - cut_tail;
    const DocPeer& dp = t.dpeer[di.peer0 + t.ch_peer[ch]];
    // atom -> row index (used by the tracker to resolve ids; reference: id_to_cursor.rs)
    u64 a0 = di.atom0 + dp.atom_base + (u32)t.op_counter[row] + cut_skip;
    for (u32 k = 0; k < len; k++) t.atom_row[a0 + k] = (u32)row;
    switch (kind) {
        case OPK_SEQ_INS:
            atomicAdd(&dc.n_ins_rows, 1u);
            atomicAdd(&dc.n_ins_atoms, len);
            break;
        case OPK_SEQ_DEL: atomicAdd(&dc.n_del_rows, 1u); break;
        case OPK_MAP_SET: case OPK_MAP_DEL: {
            atomicAdd(&dc.n_map_rows, 1u);
            u32 key = t.key_map[bi.key0 + (u32)t.op_prop[row]];
            unsigned long long pack = ((unsigned long long)lam << 32) | ((unsigned long long)dp.rank << 16) | 1ull;
            atomicMax(&t.map_best[di.mapslot0 + (u64)cidx * di.K + key], pack);
            break;
        }
        case OPK_TREE: if (!di.has_tree) di.has_tree = 1; break;   // (every writer stores the same value)
        default:
            atomicAdd(&dc.unsupported, 1u);
            atomicAdd(&di.has_unsupported, 1u);
    }
}

__global__ void k_map_winner(const DocInfo* __restrict__ docs, u64 n_rows, const __grid_constant__ BatchTables t) {
    u64 row = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    u8 kind = t.op_kind[row];
    if (kind != OPK_MAP_SET && kind != OPK_MAP_DEL) return;
    u32 ch = t.op_change[row];
    const BlockInfo& bi = t.blocks[t.ch_block[ch]];
    const DocInfo& di = docs[bi.doc];
    const DocPeer& dp = t.dpeer[di.peer0 + t.ch_peer[ch]];
    u32 key = t.key_map[bi.key0 + (u32)t.op_prop[row]];
    u64 slot = di.mapslot0 + (u64)t.op_cidx[row] * di.K + key;
    unsigned long long pack = ((unsigned long long)t.op_lamport[row] << 32) | ((unsigned long long)dp.rank << 16) | 1ull;
    if (t.map_best[slot] == pack) t.map_row[slot] = (u32)row;
}

// thread per (doc-container entry): derive tracker pool capacities from the counted rows.
__global__ void k_container_caps(DocInfo* __restrict__ docs, u32 n_docs, DocContainer* __restrict__ dcont,
                                 u32* __restrict__ cap_leaf, u32* __restrict__ cap_node,
                                 u32* __restrict__ cap_out, u32* __restrict__ cap_cvv,
                                 u32* __restrict__ doc_span_cap, u32 leaf_w) {
    u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_docs) return;
    const DocInfo& di = docs[d];
    u32 spans_total = 0;
    for (u32 c = 0; c < di.C_cap; c++) {
        u64 g = di.cid0 + c;
        u32 cl = 0, cn = 0, co = 0, cv = 0;
        if (di.code == DOC_OK && c < di.C) {
            DocContainer& dc = dcont[g];
            if ((dc.type == CT_LIST || dc.type == CT_TEXT) && (dc.n_ins_rows + dc.n_del_rows) > 0) {
                // every insert row creates one span and may split one; every delete row and every version
                // switch boundary may split two
                u64 spans = 3ull * dc.n_ins_rows + 2ull * dc.n_del_rows + 2ull * ((u64)di.n_applied + di.n_deps) + 8;
                u64 by_atoms = (u64)dc.n_ins_atoms + 2;
                if (by_atoms < spans) spans = by_atoms;
                // leaves split at leaf_w slots into halves, nodes likewise: minimum fill leaf_w / 2
                cl = (u32)(spans / (leaf_w / 2) + 4);
                cn = cl / (leaf_w / 2 - 1) + 8;
                co = (u32)spans;
                cv = di.P;
                spans_total += (u32)spans;
            }
        }
        cap_leaf[g] = cl;
        cap_node[g] = cn;
        cap_out[g] = co;
        cap_cvv[g] = cv;
        if (di.code == DOC_OK && c < di.C) {
            dcont[g].leaf_cap = cl;
            dcont[g].node_cap = cn;
            dcont[g].out_cap = co;
        }
    }
    doc_span_cap[d] = spans_total;
    docs[d].span_cap = spans_total;
}
