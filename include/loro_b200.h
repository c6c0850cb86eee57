/* loro_b200 -- C ABI of the GPU-native batched CRDT merge engine (NVIDIA H100).
 *
 * Drop-in boundary for ONE hot path of loro-dev/loro: batched `LoroDoc::import` / `import_batch` of FastUpdates blobs
 * into fresh documents (lb_import_batch*) or into documents that already hold history (lb_docset_*) -> (decode, causal
 * scan, eg-walker merge of List / Text / Map / Tree) -> deep JSON state / import status / version vector / frontiers
 * -> re-export of every document (`export(ExportMode::all_updates)`, `export(updates(from))` on demand).
 * The reference has no C FFI for this path (SURVEY.md 8b); every entry point cites the Rust interface it
 * replaces (paths relative to /root/reference):
 *
 *   lb_import_batch          crates/loro/src/lib.rs:639  LoroDoc::import(&self, &[u8]) -> Result<ImportStatus>
 *                            crates/loro/src/lib.rs:425  LoroDoc::import_batch (blobs sharing a doc_id -> one document)
 *                            crates/loro-internal/src/loro.rs:562-643 (header/checksum/mode checks first)
 *   lb_doc_status            crates/loro-internal/src/encoding.rs:226-230 ImportStatus{success,pending}
 *                            crates/loro-common/src/error.rs:8-105 (LoroError variants -> lb_doc_code)
 *   lb_doc_json              crates/loro/src/lib.rs:866  LoroDoc::get_deep_value() (serde_json text, keys sorted)
 *   lb_doc_vv                crates/loro/src/lib.rs:816  LoroDoc::oplog_vv()
 *   lb_doc_frontiers         crates/loro/src/lib.rs:881  LoroDoc::oplog_frontiers()
 *   lb_doc_export_updates    crates/loro/src/lib.rs:1235 LoroDoc::export(ExportMode::all_updates() / updates(from))
 *                            crates/loro-internal/src/encoding.rs:79-83, 350-416, oplog/change_store.rs:494-576
 *   lb_batch_export_updates  the same export for many (document, from) requests in one call
 *   lb_batch_export_updates_in_range  crates/loro-internal/src/encoding.rs:52-151 ExportMode::UpdatesInRange / updates_till
 *                            (oplog/change_store.rs:179-199), many (document, spans) requests per call
 *   lb_batch_export_json_updates  crates/loro/src/lib.rs:687-720 LoroDoc::export_json_updates(start_vv, end_vv)
 *                            (crates/loro-internal/src/loro.rs:715-751, encoding/json_schema.rs), many requests per call
 *   lb_docset_import         crates/loro/src/lib.rs:639, :425 on a document that already holds history
 *                            (crates/loro-internal/src/loro.rs:562-643, 1183-1290, oplog.rs:130-196)
 *   lb_batch_counters        crates/loro-internal/src/loro.rs:1458 len_ops / len_changes (summed over the batch)
 *   lb_import_batch_at       crates/loro-internal/src/loro.rs:1353-1433 LoroDoc::checkout(&frontiers) after the import,
 *   lb_docset_checkout       then get_deep_value() (the state at an earlier version: time travel)
 *   lb_docset_read           a stored document's get_deep_value / oplog_vv / oplog_frontiers / export, nothing imported
 *   lb_doc_attribution       who wrote the state, for the whole document: crates/loro/src/lib.rs:2644
 *                            LoroText::get_editor_at_unicode_pos, :1906 LoroList::get_id_at, :2117 LoroMap::get_last_editor,
 *                            :3046 LoroTree::get_last_move_id
 *   lb_batch_cursor_pos      crates/loro-internal/src/loro.rs:1560-1737 LoroDoc::get_cursor_pos(&Cursor) (query_pos): where
 *                            an anchored element of a Text / List lies now, for many cursors in one call
 *
 * Conventions (mirroring the reference): input buffers are borrowed for the duration of the call only;
 * outputs are owned by the batch handle until lb_batch_free; a bad blob never aborts the batch -- it yields a
 * per-document error code; checksum / mode are verified before anything else; missing dependencies are not
 * errors (they are reported as `pending`).  Thread-safe for distinct handles.
 *
 * All compute runs in hand-written CUDA kernels (sm_90a).  There is no CPU fallback: without a CUDA device
 * every entry point returns LB_ERR_NO_DEVICE.
 */
#ifndef LORO_B200_H
#define LORO_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum lb_status {
    LB_OK = 0,
    LB_ERR_INVALID_ARG = 1,
    LB_ERR_NO_DEVICE = 2,
    LB_ERR_CUDA = 3,
    LB_ERR_OOM = 4,
    LB_ERR_INTERNAL = 5,
    LB_ERR_UNSUPPORTED = 6   /* valid request the engine does not cover yet (see lb_last_error) */
} lb_status;

/* per-document result code; the LoroError variant it corresponds to is given on the right */
typedef enum lb_doc_code {
    LB_DOC_OK = 0,
    LB_DOC_ERR_DECODE = 1,          /* LoroError::DecodeError (short blob, bad magic, malformed block)  */
    LB_DOC_ERR_CHECKSUM = 2,        /* LoroError::DecodeChecksumMismatchError                            */
    LB_DOC_ERR_MODE = 3,            /* IncompatibleFutureEncodingError / ImportUnsupportedEncodingMode   */
                                    /* (a mode other than FastSnapshot 3 / FastUpdates 4)                */
    LB_DOC_ERR_CORRUPT = 4,         /* LoroError::DecodeDataCorruptionError                               */
    LB_DOC_ERR_UNSUPPORTED = 5,     /* well-formed, but outside this path: an intact FastSnapshot blob    */
                                    /* (mode 3, SURVEY 8f.1), or ops the engine does not merge yet        */
                                    /* (rich-text styles, movable list, counter), or nesting deeper than  */
                                    /* LB_MAX_NESTING                                                     */
    LB_DOC_ERR_CAPACITY = 6,        /* internal capacity bound exceeded (engine bug or adversarial input) */
    LB_DOC_ERR_FRONTIERS = 7        /* LoroError::FrontiersNotFound: a checkout id is not in the document  */
} lb_doc_code;

/* Nesting the engine covers (the reference has no bound).  A document answers LB_DOC_ERR_UNSUPPORTED when one of its
 * op values nests List / Map values more than LB_MAX_NESTING levels deep (the outermost List or Map counts; decided
 * at decode, on every path), or when its state nests child containers more than LB_MAX_NESTING levels below a root
 * container (decided while its state JSON is written, so not under LB_FLAG_NO_JSON).  The two bounds are
 * independent: a value may nest LB_MAX_NESTING levels inside a container that is itself LB_MAX_NESTING levels deep. */
#define LB_MAX_NESTING 64

typedef struct lb_blob {
    const uint8_t* ptr; /* host pointer, borrowed */
    size_t len;
    uint64_t doc_id;    /* blobs with the same doc_id are imported into ONE document (LoroDoc::import_batch,
                           crates/loro/src/lib.rs:425); documents are numbered by first appearance */
} lb_blob;

typedef struct lb_options {
    int device;          /* CUDA device ordinal */
    uint32_t flags;      /* LB_FLAG_* */
    uint32_t reserved[6];
} lb_options;
#define LB_FLAG_NO_JSON 1u      /* skip deep-value JSON materialisation */
#define LB_FLAG_KEEP_DEVICE 2u  /* keep intermediate device tables for lb_debug_* (tests) */
#define LB_FLAG_EXPORT 4u       /* also re-export every document (phase 7) for lb_doc_export_updates */
#define LB_FLAG_COMPACT 8u      /* lb_docset_import: afterwards keep each touched document as its own export (see below) */
#define LB_FLAG_ATTRIBUTION 16u /* also compute each document's attribution (phase 6b) for lb_doc_attribution */
#define LB_FLAG_CURSORS 32u     /* also keep each Text / List container's element order (after phase 5) for lb_batch_cursor_pos */

typedef struct lb_id_span {
    uint64_t peer;
    int32_t start; /* inclusive counter */
    int32_t end;   /* exclusive counter */
} lb_id_span;

typedef struct lb_import_status {
    lb_doc_code code;
    size_t n_success;
    const lb_id_span* success; /* ImportStatus.success (VersionRange) */
    size_t n_pending;
    const lb_id_span* pending; /* ImportStatus.pending */
} lb_import_status;

typedef struct lb_counters {
    uint64_t docs, docs_ok;
    uint64_t blob_bytes;
    uint64_t blocks, changes, op_rows; /* decoded */
    uint64_t atom_ops;                 /* merged ops (sum of change.atom_len of applied changes) */
    uint64_t pending_changes;
    uint64_t json_bytes;
    uint64_t state_hash;               /* xor over docs of (xxh32(json) << 32 | len): order independent */
} lb_counters;

typedef struct lb_timings { /* device time per phase in milliseconds (CUDA events on the batch stream) */
    float h2d, frame, decode, resolve, classify, integrate, materialise, d2h, total_device, reexport;
    /* algorithmic bytes of the decode phase (SURVEY.md 8d): blob bytes read + SoA bytes written */
    uint64_t decode_bytes_read, decode_bytes_written;
    /* kernels launched for this batch so far: lb_batch_timings reads it at call time, so the launches of a later
     * lb_doc_export_updates(from) show up in the next read */
    uint32_t kernel_launches;
    uint64_t export_bytes;             /* bytes written by the re-export phase */
    float tree;                        /* movable-tree phase (sort, apply, sibling lists) */
    uint32_t reserved0;
    uint64_t tree_ops;                 /* RawTreeMove rows decoded */
    /* change blocks by decode path: lane-parallel rows / staged in shared memory with the rows on one lane /
     * larger than the staging buffer (k_decode_warp.cuh) */
    uint64_t decode_fast_blocks, decode_lane_blocks, decode_unstaged_blocks;
    /* host milliseconds spent inside the device allocator while the batch was built (they are part of the wall time of
     * a step but of no device phase) and the bytes it handed out */
    float alloc_host_ms;
    uint32_t reserved1;
    uint64_t device_bytes;
    /* host wall time of the whole import call, and of its tail: from the moment the last kernel was enqueued (results
     * download, status tables) -- what a step costs beyond `total_device` */
    float host_call_ms, host_tail_ms;
    float attribution;                 /* attribution phase (LB_FLAG_ATTRIBUTION; 0 without it) */
    float cursors;                     /* import-time part of the cursor phase (LB_FLAG_CURSORS; 0 without it) */
} lb_timings;

typedef struct lb_batch lb_batch;

/* Import a batch of FastUpdates blobs from HOST memory: one fresh document per distinct doc_id (documents are
 * numbered in order of first appearance; lb_doc_count tells how many there are). */
lb_status lb_import_batch(const lb_blob* blobs, size_t n_blobs, const lb_options* opt, lb_batch** out);

/* Same, with the blobs already resident in device memory: `d_bytes` is one device buffer holding all blobs,
 * blob i occupying [offsets[i], offsets[i] + lens[i]) (HOST arrays of n_docs entries; every offset a multiple
 * of 16).  Nothing is copied host->device except these two small arrays. */
lb_status lb_import_batch_device(const uint8_t* d_bytes, const uint64_t* offsets, const uint32_t* lens,
                                 size_t n_docs, const lb_options* opt, lb_batch** out);

size_t lb_doc_count(const lb_batch* b);
lb_status lb_doc_status(const lb_batch* b, size_t doc, lb_import_status* out);
lb_status lb_doc_json(const lb_batch* b, size_t doc, const char** utf8, size_t* len);
lb_status lb_doc_vv(const lb_batch* b, size_t doc, const lb_id_span** spans, size_t* n); /* start=0,end=vv[peer] */
/* Who wrote each part of the document's state, at the version the state was built at (the latest, or the checkout's),
 * as one UTF-8 JSON object (INTEGRATION.md), canonical so that it compares byte for byte:
 *   {"peers":["<id>",...],"containers":{"<cid>":<entry>,...}}
 * `peers` are the peers of the oplog vv as decimal strings, ascending; entries name a peer by its index p there.  A
 * container is listed by its ContainerID display (full peer id) when it has an entry: root containers first by (name
 * bytes, type), then normal ones by (peer, counter).  Entries:
 *   Text / List  [[p,counter,len],...]  the ids of the visible elements in document order, in maximal runs of one peer
 *                with consecutive counters (Text counts unicode scalar values): get_editor_at_unicode_pos, get_id_at;
 *   Map          {"<key>":[p,lamport,present],...}  the winning op of every key, a delete included (present = 0), keys
 *                ascending: get_last_editor;
 *   Tree         {"<counter>@<peer>":[p,counter,alive],...}  every node the tree state holds, deleted ones included
 *                (alive = 0), by (peer, counter): [p, counter] is get_last_move_id (creation counts as a move).
 * Needs LB_FLAG_ATTRIBUTION at import (accepted by every import entry point, checkouts included; independent of
 * LB_FLAG_NO_JSON and LB_FLAG_EXPORT), otherwise LB_ERR_INVALID_ARG.  A document that failed to import (any code but
 * LB_DOC_OK) gives an empty string.  The bytes are owned by the batch. */
lb_status lb_doc_attribution(const lb_batch* b, size_t doc, const char** utf8, size_t* len);
/* ---- cursors ----------------------------------------------------------------------------------------------------------
 * LoroDoc::get_cursor_pos(&Cursor) (crates/loro-internal/src/loro.rs:1560-1737 query_pos): a Cursor anchors a place of a
 * Text or List to the element with id `id` (comments, highlights, selections, carets); the query says where that element
 * lies now.  Request i is answered in out[i]:
 *   a visible target            pos = its index (Text: unicode scalar values), side = the request's side, no update
 *                               (state.rs:1403-1433);
 *   a deleted target            pos = the visible elements before it in document order, side = Left (tracker.rs:588-619),
 *                               and an update cursor, get_cursor(pos, Left) on the current state (handler.rs:2337-2390,
 *                               :2912-2952): {no id, Left, 0} in an empty container, {no id, Right, len} when pos >= len,
 *                               otherwise {id of the visible element at pos, Left, pos};
 *   no id (has_id = 0)          pos = 0 for Left, the container's length otherwise; side = the request's side, no update;
 *   LB_CURSOR_ID_NOT_FOUND      the target was never an element of this container (another container's, a delete op's,
 *                               an id the document lacks), or a normal container the document does not have.  A root
 *                               container always exists (loro.rs:889-896): one that no op touches is empty;
 *   LB_CURSOR_CONTAINER_DELETED CannotFindRelativePosition::ContainerDeleted, kept for the mapping: the reference raises it
 *                               only for a container has_container already refused, so it is never returned;
 *   LB_ERR_INVALID_ARG          the document failed to import, or the container is not a Text or List (the reference
 *                               reaches unreachable!() for Map, Tree, Counter and MovableList), or side is not -1/0/1;
 *   LB_ERR_UNSUPPORTED          the document has code LB_DOC_ERR_UNSUPPORTED.
 * Needs LB_FLAG_CURSORS at import; lb_import_batch, lb_import_batch_device, lb_docset_import and lb_docset_read accept it.
 * lb_import_batch_at and lb_docset_checkout refuse it with LB_ERR_INVALID_ARG: on a checked-out document the reference
 * answers a visible id from the state at the checkout's version but a deleted one from the latest oplog, a mix that would
 * need both versions' orders.  The flag keeps, until lb_batch_free, one table of every span of every Text / List rope in
 * document order and one by id; without it nothing is allocated or launched.  One call uploads the requests once,
 * launches one kernel and downloads the answers once, whatever their number or documents.  The whole call fails with
 * LB_ERR_INVALID_ARG, launching nothing, for a `doc` out of range, a null pointer with a count above 0 (reqs, out, a root
 * name), or a batch imported without LB_FLAG_CURSORS; n = 0 does nothing.  Calls on one batch run one at a time. */
#define LB_CURSOR_ID_NOT_FOUND 100       /* CannotFindRelativePosition::IdNotFound */
#define LB_CURSOR_CONTAINER_DELETED 101  /* CannotFindRelativePosition::ContainerDeleted */
typedef struct lb_cursor {
    size_t doc;                 /* document index in the batch */
    /* the container: root (name bytes, type) when is_root, else normal (peer, counter, type); type as the reference
     * encodes ContainerType: 0 Map, 1 List, 2 Text, 3 Tree, 4 MovableList, 5 Counter */
    const uint8_t* name;        /* root: name bytes, borrowed for the call */
    size_t name_len;
    uint64_t peer;              /* normal: the id of the op that created it */
    int32_t counter;
    uint8_t is_root;
    uint8_t type;
    uint8_t has_id;             /* Cursor.id is Some: the target id (id_peer, id_counter) */
    int8_t side;                /* Side: -1 Left, 0 Middle, 1 Right */
    uint64_t id_peer;
    int32_t id_counter;
} lb_cursor;
typedef struct lb_cursor_result {
    int32_t status;             /* LB_OK, LB_CURSOR_ID_NOT_FOUND, LB_CURSOR_CONTAINER_DELETED, LB_ERR_INVALID_ARG,
                                   LB_ERR_UNSUPPORTED */
    int8_t side;                /* AbsolutePosition.side */
    uint8_t has_update;         /* PosQueryResult.update is Some: */
    uint8_t update_has_id;      /*   its id (update_peer, update_counter) is Some */
    int8_t update_side;
    uint64_t pos;               /* AbsolutePosition.pos */
    uint64_t update_peer;
    int32_t update_counter;
    uint32_t reserved;
    uint64_t update_origin_pos;
} lb_cursor_result;
lb_status lb_batch_cursor_pos(const lb_batch* b, const lb_cursor* reqs, size_t n, lb_cursor_result* out);
/* LoroDoc::oplog_frontiers() (crates/loro/src/lib.rs:881; version/frontiers.rs:233-246): the heads of the causal graph,
 * one span [counter, counter + 1) per head id. */
lb_status lb_doc_frontiers(const lb_batch* b, size_t doc, const lb_id_span** spans, size_t* n);
/* LoroDoc::export(ExportMode::updates(from)) of document `doc` (crates/loro/src/lib.rs:1235, encoding.rs:79-83, 350-416,
 * oplog/change_store.rs:494-528): the FastUpdates blob a fresh reference document would export after importing the same
 * input.  `from` = NULL / n_from = 0 is ExportMode::all_updates() (computed for every document at import time);
 * otherwise `from` is a version vector (one span per peer, `end` = the first counter the receiver lacks; peers not
 * listed start at 0) and the stored changes are cut there (Change::slice) -- computed on demand, the returned buffer
 * stays valid until the next from-export of the same document or lb_batch_free.  Needs LB_FLAG_EXPORT at import time.
 * LB_ERR_UNSUPPORTED: the document uses something the export phase does not cover (lb_last_error), which includes every
 * document with code LB_DOC_ERR_UNSUPPORTED; LB_ERR_INVALID_ARG: the document failed to import (any other code). */
lb_status lb_doc_export_updates(const lb_batch* b, size_t doc, const lb_id_span* from, size_t n_from,
                                const uint8_t** bytes, size_t* len);
/* Many LoroDoc::export(ExportMode::updates(from)) in one call (crates/loro/src/lib.rs:1235, encoding.rs:79-83): what a
 * sync server answers each client with, computed for all requested documents in the same device passes.  Request i
 * answers exactly what lb_doc_export_updates(b, reqs[i].doc, reqs[i].from, reqs[i].n_from, ...) answers: lb_exports_get
 * returns its status and bytes -- LB_ERR_INVALID_ARG for a document that failed to import, LB_ERR_UNSUPPORTED for one the
 * export phase does not cover -- without failing the other requests.  Requests may come in any order and name a document
 * several times.  Equal versions of one document are computed once; a version that asks for everything (n_from = 0, or
 * only peers the document lacks or counters <= 0) is the import-time all_updates blob and launches nothing; the others
 * run in rounds, round r holding the r-th distinct version of every document, so the work grows with the largest number
 * of distinct versions asked of one document, not with the number of documents.  The whole call fails with
 * LB_ERR_INVALID_ARG, and launches nothing, when a `doc` is out of range, `from` is NULL with n_from > 0, or the batch was
 * imported without LB_FLAG_EXPORT (checkout batches included).  n_reqs = 0 gives an empty result.  The bytes are host
 * memory owned by the lb_exports and stay valid until lb_exports_free, also after lb_batch_free.  Export calls on one
 * batch run one at a time. */
typedef struct lb_export_request {
    size_t doc;               /* document index in the batch */
    const lb_id_span* from;   /* version vector exactly as for lb_doc_export_updates; n_from = 0: all_updates */
    size_t n_from;
} lb_export_request;
typedef struct lb_exports lb_exports;
lb_status lb_batch_export_updates(const lb_batch* b, const lb_export_request* reqs, size_t n_reqs, lb_exports** out);
lb_status lb_exports_get(const lb_exports* e, size_t i, const uint8_t** bytes, size_t* len);
void lb_exports_free(lb_exports* e);
/* Many LoroDoc::export(ExportMode::UpdatesInRange { spans }) in one call (crates/loro-internal/src/encoding.rs:52-151,
 * oplog/change_store.rs:179-199 export_blocks_in_range): the FastUpdates blob of exactly the changes in the named id
 * spans, each stored change cut at both ends (Change::slice).  ExportMode::updates_till(vv) is one span [0, vv[p]) per
 * peer.  Spans are taken in request order.  A reversed span (start > end) covers end+1 .. start+1 (IdSpan::normalize_);
 * a span that is empty, starts below 0, or names a peer the document lacks selects nothing; one past the oplog vv is cut
 * there; a request that selects nothing gets a header-only blob.  Request order decides block boundaries: a span
 * continues the block of an earlier-listed span of its peer that ends exactly at its start, and otherwise starts a new
 * block.  The reference panics ("counter should be continuous") or stores changes twice when a peer's spans overlap, or
 * when an earlier-listed span of the peer lies below a span's start without ending there: the engine answers such a
 * request with LB_ERR_INVALID_ARG (lb_exports_get, with the reason in lb_last_error) and still answers the others.
 * Everything else follows lb_batch_export_updates: per request, LB_ERR_INVALID_ARG for a document that failed to import
 * and LB_ERR_UNSUPPORTED for one the export phase does not cover; equal span sets of one document are computed once, one
 * that selects [0, vv[p]) of every peer is the import-time blob and launches nothing, the rest run in rounds whose number
 * is the largest number of distinct span sets asked of one document; the whole call fails with LB_ERR_INVALID_ARG,
 * launching nothing, for a `doc` out of range, `spans` NULL with n_spans > 0, or a batch imported without
 * LB_FLAG_EXPORT. */
typedef struct lb_range_request {
    size_t doc;               /* document index in the batch */
    const lb_id_span* spans;  /* (peer, start, end): counters [start, end) of the peer */
    size_t n_spans;
} lb_range_request;
lb_status lb_batch_export_updates_in_range(const lb_batch* b, const lb_range_request* reqs, size_t n_reqs, lb_exports** out);
/* LoroDoc::export_json_updates(start_vv, end_vv) (crates/loro/src/lib.rs:687-720, crates/loro-internal/src/loro.rs:715-751,
 * encoding/json_schema.rs): the changes of document `doc` between two versions in the JSON schema of docs/JsonSchema.md,
 * as serde_json::to_string prints it -- UTF-8 without a terminator, returned through lb_exports_get.  Both versions are
 * refined like the reference's (a counter is clamped to the oplog vv; a peer not listed is 0, so an empty `end` exports
 * nothing); every stored change of a peer that overlaps [start, end) is listed, cut at both ends (Change::slice).  Changes
 * are ordered by lamport, equal lamports by ascending peer id (the reference leaves those in hash order); object keys of
 * nested map values are ascending.  With peer compression (the default) ids carry indices into `peers`, registered in
 * first-use order; LB_JSON_NO_PEER_COMPRESSION gives real peer ids and "peers": null.  All requests of a call run in one
 * device pass whatever their number; their text is written in chunks of bounded device size.  Errors follow
 * lb_batch_export_updates: LB_ERR_INVALID_ARG for a document that failed to import and LB_ERR_UNSUPPORTED for one the export
 * phase does not cover, per request; the whole call fails with LB_ERR_INVALID_ARG, launching nothing, for a `doc` out of
 * range, a null span pointer with a count > 0, or a batch imported without LB_FLAG_EXPORT.  n_reqs = 0 gives an empty
 * result. */
#define LB_JSON_NO_PEER_COMPRESSION 1u
typedef struct lb_json_request {
    size_t doc;
    const lb_id_span* start; size_t n_start;   /* start_vv, spans as for lb_export_request.from */
    const lb_id_span* end;   size_t n_end;     /* end_vv: a peer not listed ends at 0 */
    uint32_t flags;                            /* LB_JSON_NO_PEER_COMPRESSION */
} lb_json_request;
lb_status lb_batch_export_json_updates(const lb_batch* b, const lb_json_request* reqs, size_t n_reqs, lb_exports** out);
lb_status lb_batch_counters(const lb_batch* b, lb_counters* out);
lb_status lb_batch_timings(const lb_batch* b, lb_timings* out);
const char* lb_last_error(void); /* thread-local, human readable */
/* Device blocks that lived until lb_batch_free are kept (per device, by size class, at most LB_DEV_CACHE_GB gigabytes,
 * default 85 % of the device's memory) for the next batch of similar shape; this gives them back to the driver. */
lb_status lb_device_trim(int device);

/* One process per GPU: pin the calling thread -- and the staging / download threads the engine creates from it -- to
 * the CPUs of the NUMA node `device` is attached to (sysfs).  Call before building the input buffers so that they,
 * the pinned staging ring and the gather threads all sit next to the GPU.  LB_ERR_UNSUPPORTED: topology unknown. */
lb_status lb_numa_bind(int device);
void lb_batch_free(lb_batch* b);

/* ---- persistent documents: imports against an EXISTING document state ------------------------------------------------
 * LoroDoc::import / import_batch on a document that already holds history (crates/loro/src/lib.rs:639, :425;
 * crates/loro-internal/src/loro.rs:562-643, 1183-1290; oplog.rs:130-196: changes the document knows are skipped or
 * trimmed, pending changes wait in the oplog until a later import brings their dependencies).
 * A docset keeps, per doc_id, the document's change store in wire form IN DEVICE MEMORY: the update blobs it has
 * imported, in order (what the reference's ChangeStore keeps are encoded blocks too, change_store.rs:60-110).
 * lb_docset_import lays the stored blobs of every touched document in front of the new ones (device-to-device) and
 * replays the document; the batch it returns answers exactly like the reference's import on the existing document:
 *   lb_doc_status    ImportStatus of THIS import: success = what the new blobs added (a change the document already
 *                    held is not reported, a stored pending change released by this import is), pending = what the
 *                    new blobs parked;
 *   lb_doc_json / lb_doc_vv / lb_doc_frontiers / lb_doc_export_updates    the document after the import.
 * Several blobs with one doc_id in one call = import_batch on that document (sorted by mode, then number of changes
 * descending, among the new blobs).  A document whose import fails (checksum, decode error, ...) keeps its earlier
 * state, like the reference (loro.rs:584: checked before any state change).
 * LB_FLAG_COMPACT in `opt->flags`: after this import every touched document without pending changes is replaced by a
 * fresh document that imported its own export -- `fresh.import(doc.export(all_updates))`, the way a host drops
 * redundant history; the stored form shrinks to one blob.  State, vv and frontiers are unaffected; later exports equal
 * those of a reference document that was re-created the same way (the op segmentation of an export depends on which
 * blob brought which piece of a change, so they may differ by a few bytes from an uncompacted document's).
 * The engine merges by replaying the
 * document's whole history, not from the common ancestor of the two versions (dag.rs:488-667): same results, the
 * cost of an import grows with the history (SURVEY 8a row a12; DESIGN.md section 9).
 * One docset serves one device; calls on the same docset are serialised.  LB_FLAG_EXPORT is implied. */
typedef struct lb_docset lb_docset;
lb_status lb_docset_new(const lb_options* opt, lb_docset** out);
lb_status lb_docset_import(lb_docset* set, const lb_blob* blobs, size_t n_blobs, const lb_options* opt, lb_batch** out);
size_t lb_docset_doc_count(const lb_docset* set);
uint64_t lb_docset_stored_bytes(const lb_docset* set);   /* device bytes of the stored documents */
void lb_docset_free(lb_docset* set);

/* ---- checkout: a document's state at an earlier version -----------------------------------------------------------
 * LoroDoc::checkout(&frontiers) followed by get_deep_value() (crates/loro-internal/src/loro.rs:1353-1433).  The state at
 * Frontiers F is built from every atom in the causal closure of F and from nothing else: a change that straddles the
 * version is cut inside, its op under the cut inside the op.  Every id of F must be an atom the document holds (not an
 * unknown peer, not a counter at or past the oplog vv, not inside a pending change), otherwise the document's code is
 * LB_DOC_ERR_FRONTIERS (LoroError::FrontiersNotFound, loro.rs:1394-1410).  Redundant ids are allowed; n_frontiers = 0 is
 * the empty version.  Every root container the document has registered is listed, with or without ops inside F
 * (state.rs:894-924).  What a result handle answers for a requested document:
 *   lb_doc_json                  get_deep_value() after the checkout;
 *   lb_doc_status                the import's code and spans (LB_DOC_ERR_FRONTIERS when the import succeeded but F is
 *                                not in the document; LB_DOC_ERR_UNSUPPORTED is decided over the whole applied history);
 *   lb_doc_vv / lb_doc_frontiers the OPLOG's version vector and frontiers (the state's version is the request);
 *   lb_doc_export_updates        LB_ERR_INVALID_ARG: a checked-out document is not exported. */
typedef struct lb_version {
    uint64_t doc_id;                 /* document doc_id at Frontiers `frontiers`: one span [counter, counter + 1) per id, */
    const lb_id_span* frontiers;     /* the form lb_doc_frontiers returns; n_frontiers = 0 is the empty version            */
    size_t n_frontiers;
} lb_version;
/* lb_import_batch(blobs), then checkout(F) of every document named in `at` (documents are numbered as in
 * lb_import_batch).  A document that is not named stays at the latest version and answers byte for byte like
 * lb_import_batch; naming it with n_frontiers = 0 asks for the empty version.  LB_ERR_INVALID_ARG: a doc_id named twice or
 * carried by no blob, null frontiers with n_frontiers > 0, LB_FLAG_EXPORT or LB_FLAG_COMPACT in the flags. */
lb_status lb_import_batch_at(const lb_blob* blobs, size_t n_blobs, const lb_version* at, size_t n_at,
                             const lb_options* opt, lb_batch** out);
/* One document per request, in request order: the stored document doc_id at Frontiers F (a doc_id may repeat, at different
 * versions; one the set has never seen is an empty document).  The status spans are empty: nothing is imported.  The
 * docset is not modified.  LB_ERR_INVALID_ARG: null frontiers with n_frontiers > 0, LB_FLAG_EXPORT or LB_FLAG_COMPACT. */
lb_status lb_docset_checkout(lb_docset* set, const lb_version* at, size_t n_at, const lb_options* opt, lb_batch** out);

/* ---- reading stored documents ---------------------------------------------------------------------------------------
 * The stored documents as they are, without importing anything (a sync server answering a client that connects with
 * nothing to send): one document per doc_id, in the order given, each holding its stored blobs laid out exactly as
 * lb_docset_import lays them and no new blob; an id the set has never seen is an empty document.  The batch is imported
 * with LB_FLAG_EXPORT: lb_doc_json (get_deep_value, crates/loro/src/lib.rs:866), lb_doc_vv, lb_doc_frontiers,
 * lb_doc_export_updates and lb_batch_export_updates (crates/loro/src/lib.rs:1235, encoding.rs:79-83) answer for the
 * stored document; lb_doc_status gives the document's code with empty spans (nothing was imported).  LB_FLAG_NO_JSON is
 * honoured.  The docset is not modified.  LB_ERR_INVALID_ARG: a doc_id listed twice, LB_FLAG_COMPACT. */
lb_status lb_docset_read(lb_docset* set, const uint64_t* doc_ids, size_t n, const lb_options* opt, lb_batch** out);

/* test hooks (need LB_FLAG_KEEP_DEVICE): copy one decoded SoA table to the host.
 * name in {"op_cid","op_prop","op_vtype","op_len","op_counter","ch_counter","ch_len","ch_lamport",
 *          "ch_ts","dep_peer","dep_counter","blk_doc","blk_nchanges"}; returns element count. */
lb_status lb_debug_table(const lb_batch* b, const char* name, void* dst, size_t dst_bytes, size_t* n_elems,
                         size_t* elem_size);

#ifdef __cplusplus
}
#endif
#endif
