/* Plain-C caller of libloro_b200.so: a batch import of fresh documents, then the same documents kept in a docset and
 * updated in place.  This is the shape of the binding a loro host adds (INTEGRATION.md shows the Rust `extern "C"`
 * equivalent).  Build:  gcc -std=c99 -Iinclude examples/c/import_and_docset.c -Lloro_b200 -lloro_b200 -o demo
 * Run (needs a CUDA device):  ./demo update1.bin update2.bin   -- both blobs are imported into ONE document. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "loro_b200.h"

static uint8_t* read_file(const char* path, size_t* len) {
    FILE* f = fopen(path, "rb");
    if (!f) return NULL;
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    uint8_t* p = (uint8_t*)malloc((size_t)n + 1);
    if (p && fread(p, 1, (size_t)n, f) != (size_t)n) { free(p); p = NULL; }
    fclose(f);
    *len = (size_t)n;
    return p;
}

static void print_doc(const lb_batch* b, size_t doc) {
    lb_import_status st;
    if (lb_doc_status(b, doc, &st) != LB_OK) return;
    printf("document %zu: code %d, %zu peers imported, %zu pending\n", doc, (int)st.code, st.n_success, st.n_pending);
    for (size_t k = 0; k < st.n_success; k++)
        printf("  success peer %llu [%d, %d)\n", (unsigned long long)st.success[k].peer, st.success[k].start, st.success[k].end);
    const char* json;
    size_t n;
    if (st.code == LB_DOC_OK && lb_doc_json(b, doc, &json, &n) == LB_OK) printf("  state: %.*s\n", (int)(n < 200 ? n : 200), json);
    const uint8_t* bytes;
    if (st.code == LB_DOC_OK && lb_doc_export_updates(b, doc, NULL, 0, &bytes, &n) == LB_OK) printf("  export(all_updates): %zu bytes\n", n);
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: %s update.bin [more updates of the same document ...]\n", argv[0]); return 2; }
    lb_options opt;
    memset(&opt, 0, sizeof(opt));
    opt.flags = LB_FLAG_EXPORT | LB_FLAG_CURSORS;
    /* 1. LoroDoc::import_batch into a fresh document: every blob carries the same doc_id */
    size_t n = (size_t)argc - 1;
    lb_blob* blobs = (lb_blob*)calloc(n, sizeof(lb_blob));
    for (size_t i = 0; i < n; i++) {
        blobs[i].ptr = read_file(argv[i + 1], &blobs[i].len);
        blobs[i].doc_id = 1;
        if (!blobs[i].ptr) { fprintf(stderr, "cannot read %s\n", argv[i + 1]); return 2; }
    }
    lb_batch* b = NULL;
    lb_status rc = lb_import_batch(blobs, n, &opt, &b);
    if (rc != LB_OK) { fprintf(stderr, "lb_import_batch: %d (%s)\n", (int)rc, lb_last_error()); return 1; }
    print_doc(b, 0);
    /* LoroDoc::get_cursor_pos: a cursor at the end of the root Text "text" (no id, Side::Right) lies at its length */
    lb_cursor cur;
    memset(&cur, 0, sizeof(cur));
    cur.doc = 0;
    cur.name = (const uint8_t*)"text";
    cur.name_len = 4;
    cur.is_root = 1;
    cur.type = 2;   /* Text */
    cur.side = 1;
    lb_cursor_result res;
    if (lb_batch_cursor_pos(b, &cur, 1, &res) != LB_OK) { fprintf(stderr, "lb_batch_cursor_pos: %s\n", lb_last_error()); return 1; }
    printf("  cursor at the end of text: status %d, pos %llu\n", (int)res.status, (unsigned long long)res.pos);
    lb_batch_free(b);
    /* 2. the same updates one call at a time against a document that lives in device memory between the calls */
    lb_docset* set = NULL;
    if (lb_docset_new(&opt, &set) != LB_OK) { fprintf(stderr, "lb_docset_new: %s\n", lb_last_error()); return 1; }
    for (size_t i = 0; i < n; i++) {
        if (lb_docset_import(set, &blobs[i], 1, &opt, &b) != LB_OK) { fprintf(stderr, "lb_docset_import: %s\n", lb_last_error()); return 1; }
        print_doc(b, 0);   /* the status of THIS import, the document after it */
        lb_batch_free(b);
    }
    printf("docset: %zu document(s), %llu bytes stored on the device\n", lb_docset_doc_count(set),
           (unsigned long long)lb_docset_stored_bytes(set));
    lb_docset_free(set);
    for (size_t i = 0; i < n; i++) free((void*)blobs[i].ptr);
    free(blobs);
    return 0;
}
