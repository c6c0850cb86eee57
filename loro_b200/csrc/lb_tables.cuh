// loro_b200 -- the batch's device tables, one definition for every phase.
//
// Each table has exactly one name.  The fields are grouped by the phase that writes them; a kernel reads what the
// earlier phases wrote through the same struct, which the host fills in place (engine.cu pipeline()).  Tables a batch
// does not need stay null (the tree tables without tree ops, the epochs of single-blob documents, phase 7 without
// LB_FLAG_EXPORT).  Kernels take it as `const __grid_constant__ BatchTables`, so helpers can hold a reference to it
// without a copy to local memory.
#pragma once
#include "lb_defs.h"

struct XDoc;   // k_export.cuh
struct XSpan {   // counters [start, end) of one peer to export; fresh = 1: the span starts a new block in the export store
    i32 start, end;
    u32 fresh, pad;
};

struct BatchTables {
    // ---- input and phase 1 (frame)
    const u8* bytes;          // the batch byte buffer
    BlockInfo* blocks;
    // ---- phase 2: decode (k_decode.cuh), block-local index spaces
    u64* peer_id;             // block-local peer tables
    u64* key_off; u32* key_len;   // keys (block-local arena; the keys of nested map values index it too)
    u8* cid_root; u8* cid_type; u32* cid_peer_idx; i32* cid_koc;  // cids (block-local arena) ; koc: key idx or counter
    u32* ch_block; i32* ch_counter; u32* ch_len;
    u32* ch_lamport_wire;     // lamport as read from the block (ch_lamport: recomputed by phase 3)
    i64* ch_ts; u64* ch_msg_off; u32* ch_msg_len;
    u64* ch_dep0; u32* ch_ndeps; u8* ch_dep_self; u64* ch_op0; u32* ch_nops;
    u32* dep_peer_idx; i32* dep_counter;   // deps (other peers)
    // op rows
    u32* op_cid; i32* op_prop; u8* op_vtype; u32* op_len; i32* op_counter; u32* op_change;
    u64* op_val_off; u32* op_val_len;      // value payloads
    u32* op_del;              // index into the del tables for DeleteSeq rows, into tr_* for RawTreeMove rows
    u32* del_peer_idx; i32* del_counter; i32* del_len;   // delete start ids
    // fractional indexes (expanded) + decoded RawTreeMove fields
    u64* pos_off; u32* pos_len; u8* pos_pool;
    u32* tr_target_peer; i32* tr_target_ctr; u8* tr_parent_kind; u32* tr_parent_peer; i32* tr_parent_ctr; u32* tr_pos;
    unsigned long long* dw_stats;   // [0] blocks decoded lane-parallel, [1] staged but rows on one lane, [2] not staged
    // ---- phase 3: resolve (k_resolve.cuh).  Index spaces: peers <-> block peer entries, containers <-> block cid
    // entries, keys <-> block key entries, changes <-> batch-wide change index
    DocPeer* dpeer; u32* peer_map;
    DocContainer* dcont; u32* cid_map;
    u64* dkey_off; u32* dkey_len; u32* key_map;
    u32* blk_order;      // per doc: its blocks sorted by (peer, counter_start)
    u32* ch_order;       // per doc: changes grouped by peer, counter order (batch-wide change ids): every COPY
    u32* ch_aorder;      // same grouping: the peer's APPLIED copies in the order they were applied (their applied ranges
                         // [counter + trim, counter + len) are disjoint and ascending), then the copies that were not;
                         // this is the order every later phase walks (tracker version switches, change store)
    u16* ch_peer;        // doc peer idx of each change
    u8* ch_applied;
    u32* ch_lamport;     // recomputed lamport
    u32* ch_walk;        // per doc: applied changes in replay order
    i32* ch_vv;          // per doc: n_changes * P
    u32* ch_pos;         // per change: its position in the doc's ch_order (= row of ch_vv)
    u32* ch_trim;        // per change: leading atoms the document already had when the change arrived
                         // (OpLog::trim_the_known_part_of_change, oplog.rs:181-196: the rest is applied as a slice)
    u32* ch_epoch;       // per change COPY of a multi-blob document: the rank of the blob during whose import the reference
                         // can first apply it (its own blob, or the later one that brings its last missing dependency:
                         // blobs of a document are imported one after the other, loro.rs:1183-1290, and parked changes wait
                         // in the pending store, pending_changes.rs); bit 31: in that blob's FIRST pass
                         // (import_changes_to_oplog) rather than by its try_apply_pending
    i32* ch_maxend;      // per position of the per-peer change lists: highest counter end among the entries up to there
    u32* head_lamport;   // per doc peer: lamport of the first atom of the copy at the status pass's cursor
    // ---- phase 4: classify + map LWW (k_classify.cuh)
    u64* tr_key;         // (lamport << 32 | peer rank << 16): the total order of a tree's ops (diff_calc/tree.rs:445-452),
                         // ~0 for ops that are not applied
    uint4* tr_ids;       // x = target peer (document level), y = target counter, z = parent kind | parent peer << 2, w = parent counter
    uint4* tr_rec;       // x = target atom (document-relative), y = parent atom | TREE_ROOT | TREE_DELETED, z = position, w = row
    u8* op_kind; u32* op_cidx; u32* op_lamport;
    uint4* op_rec; u32* op_aux;   // compact records for the tracker (layout: k_seq.cuh REC_*)
    u32* atom_row;       // per doc: atom -> op row (batch-wide row index, 32-bit)
    unsigned long long* map_best;  // per (doc, container, key): max packed (lamport<<32 | rank<<16 | 1)
    u32* map_row;        // winner row per slot
    // ---- phase 5: sequence integration (k_seq.cuh): final visible runs per container (DocContainer::out0)
    u32* out_row; u32* out_off; u32* out_len;
    // ---- phase 5b: movable trees (k_tree.cuh)
    u64* ts_key; u32* ts_val; // sort space, one entry per tree op
    uint4* ts_rec;            // the records in apply order (w = 0xFFFFFFFF from the first op that is not applied)
    // per document: S = atom_total + C slots starting at DocInfo::tree0.  Slots [0, atom_total) are nodes, slot
    // atom_total + c is the root of tree container c.
    u32* tn_parent;           // [node] TREE_UNEXIST | TREE_ROOT | TREE_DELETED | parent node
    u32* tn_move;             // [node] tree op of the last effective move (position, lamport, peer of the node)
    u32* tn_base;             // [slot] first child in tn_child
    u32* tn_cnt;              // [slot] number of children
    u32* tn_sib;              // [node] index among its siblings
    u64* ns_key;              // [slot] sort key: parent slot << 32 | first four position bytes; after the sort the space holds
                              //        tn_sub (JSON bytes of the subtree, [slot]) and tn_rel (offset among siblings, [node])
    u32* tn_child;            // [node] after the sort: nodes grouped by parent slot, in sibling order
    // hierarchy JSON layout (k_state.cuh writes the nodes lane-parallel when no node has a meta map with content)
    u32* tn_root;             // [node] root slot of the tree the node is alive in, TREE_UNEXIST when dead
    u32* tn_aopen;            // [node] offset of the node's `{"children":[` inside its container's JSON
    u32* tn_aclose;           // [node] offset of the part after its children
    // ---- phase 7: re-export (k_export.cuh)
    u32* pos_rank;     // per position entry: dense rank of its bytes among the document's positions
    u32* pos_rep;      // per (document position base + rank): one entry holding those bytes
    u64* ps_key; u32* ps_val;   // sort space of k_exp_posrank
    // per row
    uint4* x_rec;      // resolved op record per row (xop_pack): kind | reversed | container, counter, prop, arena start / target counter
    u32* r_bytes;      // text rows: payload bytes
    u8* r_flag;        // XF_*
    // per change
    u32* ch_nseg;      // segments the change enters the store as (0 = not applied)
    u32* ch_novf;      // nseg - 1 (scan input): only split changes need slots beyond their own
    // changes whose split cuts an op (Op::slice, list_op.rs:603-658) get SYNTHETIC rows: one per source row or slice,
    // addressed as row = n_rows + ch_syn0[ch] + i; every row accessor understands both spaces
    u32* ch_syn; u64* ch_syn0; u64 n_rows;
    u32 has_syn;       // any synthetic row in the batch (uniform: the common batch never leaves the decoded rows)
    uint4* s_rec; u32* s_len; u32* s_bytes; u8* s_flag; u64* s_voff; u32* s_vlen; u32* s_aux;
    u64 n_changes;     // segment q of change ch lives at q == 0 ? ch : n_changes + ch_seg0[ch] + q - 1
    u32* ch_aval; u32* ch_astr; u64* ch_aval0; u64* ch_astr0;   // arena sums per change + their scans
    u64* ch_seg0;      // scan of ch_novf
    // per segment
    u32* sg_src; u32* sg_r0; u32* sg_from; u32* sg_atoms; u32* sg_est; u32* sg_nmops; u32* sg_ndel; u32* sg_nrows; u32* sg_last_head;
    u32* sg_skip;      // atoms of the segment's first row the document already had (import-side trim, k_doc_causal)
    // final changes (same index space: a document never ends up with more changes than segments)
    u32* fc_src; u32* fc_pos; u32* fc_r0; u32* fc_from; u32* fc_atoms; u32* fc_nrows; u32* fc_ndel; u8* fc_block;
    u32* fc_skip;      // atoms of the change's first row that lie before its span (Change::slice at the front)
    u32* fc_tail;      // atoms of the change's last row that lie at or past the end of its span (Change::slice at the end)
    u32* fc_est;       // the store's size estimate of the change's ops (sizes the staging slot of its block)
    // export of chosen id spans on demand (lb_batch_export_updates, lb_batch_export_updates_in_range): x_req[d] != 0
    // marks the documents of one round (null: every document, the import-time export); the spans of doc peer slot s are
    // x_spans[x_span0[s] .. x_span0[s + 1]), disjoint and sorted by start (null: [0, vv) for every peer).  updates(from)
    // is one span [from, vv) per peer (encoding.rs:79-83, change_store.rs:494-528); UpdatesInRange is the caller's spans
    // (change_store.rs:179-199).  export_round sets these on a copy of the batch's struct.
    const u8* x_req; const u32* x_span0; const XSpan* x_spans;
    XDoc* xdoc;
    // ---- checkout (k_checkout.cuh), written after the causal scan, read by phases 4 and 5 (last, so that the layout of
    // every other field is the same with or without it)
    i32* ck_end;         // per doc peer: the version the state is built at: atoms at or past it are cut; end_counter for
                         // documents without a request.  Null when the batch has no checkout request
};
