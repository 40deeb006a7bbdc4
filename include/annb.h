/*
 * annb.h -- C ABI of libannlite_b200.so: the H100 (sm_90a) implementation of AnnLite's
 * PQ-ADC / PQ-HNSW search path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point below replaces one
 * native call the reference makes through `annlite.pq_bind` (Cython) or
 * `annlite.hnsw_bind.Index` (pybind11); the reference interface it stands in for is cited as
 * file:line relative to the reference tree.  Plain pointers and sizes only -- no torch, no
 * C++ types.  All functions return 0 on success and a negative ANNB_E* code on failure;
 * annb_last_error() returns the message for the calling thread (the strings mirror the
 * reference's exception texts so the Python shim can raise the same exceptions).
 *
 * Memory spaces: every data pointer is accompanied by (or covered by) a `space` argument:
 * ANNB_HOST = ordinary host memory (numpy), ANNB_DEVICE = device memory on the handle's GPU
 * (e.g. torch `tensor.data_ptr()`).  Host pointers are borrowed for the duration of the call
 * only.  Work is enqueued on the handle's own CUDA stream; calls taking host output buffers
 * synchronise that stream before returning, calls with device outputs return asynchronously
 * (use annb_sync / annb_stream).
 *
 * There is no CPU fallback: every compute entry point fails with ANNB_ENODEVICE when no CUDA
 * device is usable.
 */
#ifndef ANNB_H_
#define ANNB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ANNB_VERSION 100 /* 0.1.0 */

#if defined(__GNUC__)
#define ANNB_API __attribute__((visibility("default")))
#else
#define ANNB_API
#endif

/* status codes */
#define ANNB_OK 0
#define ANNB_EINVAL (-1)     /* bad argument / wrong dimensionality                              */
#define ANNB_ENODEVICE (-2)  /* no usable CUDA device (there is no CPU path)                     */
#define ANNB_ECUDA (-3)      /* CUDA runtime error (message has the cudaError string)            */
#define ANNB_ENOMEM (-4)
#define ANNB_ESTATE (-5)     /* call order: codebook / codes / graph not set                      */
#define ANNB_EFEWRESULTS (-6)/* a query found < k results: hnsw_bindings.cpp:342-345 / :461-464   */
#define ANNB_EIO (-7)        /* "Cannot open file" / "Index seems to be corrupted or unsupported" */
#define ANNB_ECAPACITY (-8)  /* "The number of elements exceeds the specified limit" hnswalg.h:1133 */
#define ANNB_ENOTFOUND (-9)  /* "Label not found" hnswalg.h:878-880                               */
#define ANNB_ELIMIT (-10)    /* outside this build's limits (ef > ANNB_MAX_EF, code width ...)    */

#define ANNB_HOST 0
#define ANNB_DEVICE 1

/* metric: annlite/enums.py:25-28 -> space names 'l2' / 'ip' / 'cosine' (hnsw/index.py:196-202) */
#define ANNB_METRIC_L2 0
#define ANNB_METRIC_IP 1
#define ANNB_METRIC_COSINE 2

#define ANNB_MAX_EF 512 /* top-candidate list lives in registers: 16 entries x 32 lanes */

typedef struct annb_index annb_index_t;

/* ---- library / error -------------------------------------------------------------------- */
ANNB_API int annb_version(void);
ANNB_API const char *annb_last_error(void);
ANNB_API int annb_device_count(void);

/* ---- lifetime --------------------------------------------------------------------------- */

/* Index(space, dim) + _loadPQ geometry (hnsw_bindings.cpp:87-112, :851-928).
 * dim == n_subvectors * d_subvector is enforced (:883-891); code width follows n_clusters:
 * <=256 -> u8, <=65536 -> u16 (:909-927; u32 codes are rejected with ANNB_ELIMIT).
 * device >= 0 selects the GPU.  device == -1 creates a HOST-ONLY handle that can hold, load, save and
 * extend (annb_add_items_with_tables) a graph but cannot compute anything: every kernel-backed entry
 * point returns ANNB_ENODEVICE on it.  It exists for tooling and CPU-side tests of the container. */
ANNB_API int annb_create(int device, int metric, int dim, int n_subvectors, int n_clusters,
                annb_index_t **out);
ANNB_API int annb_destroy(annb_index_t *h);

/* The codebook a trained PQCodec hands to _loadPQ via get_codebook() (hnsw_bindings.cpp:892-905,
 * annlite/core/codec/pq.py:231-237): (n_subvectors, n_clusters, d_subvector) fp32, C-contiguous. */
ANNB_API int annb_set_codebook(annb_index_t *h, const float *codebook, int space);

/* cudaStream_t of the handle as an integer (for torch.cuda.ExternalStream) and a blocking sync. */
ANNB_API int annb_stream(annb_index_t *h, uint64_t *stream_out);
ANNB_API int annb_sync(annb_index_t *h);

/* ---- K1: ADC tables -------------------------------------------------------------------- */

/* pq_bind.batch_precompute_adc_table (bindings/pq_bindings.pyx:149-210; single query :85-145),
 * pq_bind.batch_precompute_adc_table_ip (:214-274) followed by the `1/n_clusters - .` epilogue of
 * PQCodec.get_dist_mat (annlite/core/codec/pq.py:293-325).  The metric of the handle selects the
 * formula.  queries: (B, dim) fp32; out: (B, n_subvectors, n_clusters) fp32.
 * normalize != 0 applies annlite.math.l2_normalize (annlite/math.py:6-18) to each query first,
 * `normalize` times (HnswIndex.search normalises twice for COSINE: hnsw/index.py:28-29 and
 * pq.py:309-310).  Arithmetic order and rounding match the reference (sequential over j,
 * no FMA contraction). */
ANNB_API int annb_adc_table(annb_index_t *h, const float *queries, int q_space, int64_t B, int normalize,
                   float *out, int out_space);

/* ---- K2: exhaustive ADC scan ------------------------------------------------------------ */

/* The flat code matrix PQIndex keeps in `_data` (annlite/core/index/pq_index.py:25-27,
 * flat_index.py:47-56): (n, n_subvectors) u8/u16.  Independent of the HNSW graph. */
ANNB_API int annb_set_codes(annb_index_t *h, const void *codes, int space, int64_t n);

/* pq_bind.dist_pqcodes_to_codebooks (bindings/pq_bindings.pyx:52-80): one (M,Ks) table against
 * all n codes -> n fp32 distances. */
ANNB_API int annb_scan(annb_index_t *h, const float *table, int t_space, float *out_dists, int out_space);

/* PQIndex.search for a batch (pq_index.py:29-56 + annlite/math.py:94-120): per query the k
 * smallest ADC distances over the code matrix, ascending; ties ordered by row index.
 * `tables` may be NULL, in which case they are built from `queries` with K1 (fused path).
 * ids: (B,k) int64 row indices, dists: (B,k) fp32 (squared L2 / raw IP form, no sqrt). */
ANNB_API int annb_scan_topk(annb_index_t *h, const float *queries, const float *tables, int in_space,
                   int64_t B, int k, int64_t *ids, float *dists, int out_space);

/* ---- HNSW graph: import / export / build ------------------------------------------------- */

/* Index.init_index(max_elements, M, ef_construction, random_seed) (hnsw_bindings.cpp:144-163,
 * :941-943; hnswalg.h:27-69).  Creates an empty graph with the reference's memory layout. */
ANNB_API int annb_init_graph(annb_index_t *h, int64_t max_elements, int M, int ef_construction,
                    uint64_t random_seed);

/* Index.load_index(path, max_elements) / Index.save_index(path): hnswlib's binary format
 * (hnswalg.h:708-736, :738-846) -- files are interchangeable with the reference. */
ANNB_API int annb_load_index(annb_index_t *h, const char *path, int64_t max_elements);
ANNB_API int annb_save_index(annb_index_t *h, const char *path);

/* Index.__setstate__ / createFromParams + setAnnData (hnsw_bindings.cpp:691-841): adopt a graph
 * given as the raw arrays of the reference's pickle dict. */
ANNB_API int annb_set_graph(annb_index_t *h, const uint8_t *data_level0, uint64_t data_level0_bytes,
                   uint64_t size_data_per_element, uint64_t offset_data, uint64_t label_offset,
                   const uint8_t *link_lists, uint64_t link_lists_bytes, const int32_t *element_levels,
                   int64_t n_element_levels, uint64_t size_links_per_element,
                   int64_t cur_element_count, int64_t max_elements, int32_t max_level,
                   uint32_t enterpoint_node, int max_M, int max_M0, int M, int ef_construction,
                   double mult);
/* The three array extents (bytes of data_level0 / link_lists, entries of element_levels) are what the
 * caller really holds; the state is rejected (ANNB_EINVAL) if cur_element_count or the levels ask for
 * more, and then checked structurally like a loaded file. */

/* Index.__getstate__ (hnsw_bindings.cpp:549-671): sizes first, then copy-out. */
ANNB_API int annb_graph_info(annb_index_t *h, int64_t *cur_element_count, int64_t *max_elements,
                    uint64_t *size_data_per_element, uint64_t *link_lists_bytes, int32_t *max_level,
                    uint32_t *enterpoint_node, int *max_M, int *max_M0, int *M, int *ef_construction,
                    double *mult);
ANNB_API int annb_get_graph(annb_index_t *h, uint8_t *data_level0, uint8_t *link_lists, int32_t *element_levels);

/* Index.add_items(data, ids, num_threads, dtables) (hnsw_bindings.cpp:216-300 -> hnswalg.h:1108-1235).
 * `vectors`: (n, dim) fp32 rows (already l2-normalised by the caller for COSINE, as pre_process
 * does); the library encodes them (PQCodec.encode, pq.py:158-177) unless `codes` is given, builds
 * each row's ADC table on the fly (the reference materialises (n,M,Ks) tables; this does not)
 * and inserts with the reference's algorithm, including its PQ-mode neighbour heuristic
 * (SURVEY.md section 0.2).  num_threads == 1 reproduces the reference's single-threaded graph
 * bit for bit; > 1 inserts concurrently like ParallelFor (hnsw_bindings.cpp:24-77). */
ANNB_API int annb_add_items(annb_index_t *h, const float *vectors, const void *codes, const uint64_t *labels,
                   int64_t n, int num_threads);

/* The literal shape of Index.add_items(data=codes, ids, num_threads, dtables) (hnsw_bindings.cpp:286-300):
 * caller-supplied PQ codes (n, n_subvectors) and the materialised (n, n_subvectors, n_clusters) fp32
 * tables, both host memory.  Kept for call-site compatibility; annb_add_items is the path that
 * does not need O(n*M*Ks) host memory. */
ANNB_API int annb_add_items_with_tables(annb_index_t *h, const void *codes, const float *tables,
                               const uint64_t *labels, int64_t n, int num_threads);

/* PQCodec.encode (pq.py:158-177): nearest codeword per subspace, first minimum. (n,dim)->(n,M). */
ANNB_API int annb_encode(annb_index_t *h, const float *vectors, int v_space, int64_t n, void *codes, int c_space);

ANNB_API int annb_resize_index(annb_index_t *h, int64_t new_max_elements); /* hnswalg.h:680-706           */
ANNB_API int annb_mark_deleted(annb_index_t *h, uint64_t label);           /* hnswalg.h:875-902           */
ANNB_API int annb_unmark_deleted(annb_index_t *h, uint64_t label);         /* hnswalg.h:908-934           */
ANNB_API int annb_element_count(annb_index_t *h, int64_t *out);            /* hnsw_bindings.cpp:987-992   */
/* Index.get_ids_list (hnsw_bindings.cpp:539-547): labels in internal-id order. */
ANNB_API int annb_get_labels(annb_index_t *h, uint64_t *labels_out, int64_t cap);
/* Index.get_items(ids) (hnsw_bindings.cpp:518-537): stored PQ codes of the given labels. */
ANNB_API int annb_get_codes(annb_index_t *h, const uint64_t *labels, int64_t n, void *codes_out);

/* ---- K3: HNSW search ---------------------------------------------------------------------- */

/* Index.knn_query(data, k, num_threads, dtables) (hnsw_bindings.cpp:303-391 -> hnswalg.h:1237-1295)
 * and Index.knn_query_with_filter(data, filters, k, num_threads, dtables) (:393-516 ->
 * hnswalg.h:1297-1361).
 *   queries / tables : exactly one non-NULL.  `tables` = the (B,M,Ks) `dtables` argument;
 *                      `queries` = (B,dim) fp32, tables are then built on the device (K1) with
 *                      `normalize` rounds of l2_normalize first.
 *   ef               : Index.set_ef value; the search uses max(ef, k) (hnswalg.h:1279).
 *   filter_labels    : NULL = knn_query; else the `filters` array of allowed labels (host or
 *                      device per `filter_space`), n_filter entries.  Membership is exact (the
 *                      reference's binary-fuse-16 filter approximates the same set).
 *   labels_out       : (B,k) uint64, dists_out: (B,k) fp32, rows ascending by (dist, label) --
 *                      the order produced by the unload loop at hnsw_bindings.cpp:346-351.
 *   stats_out        : optional (B,3) int64 {hops, neighbours listed, distances computed}:
 *                      metric_hops / metric_distance_computations of hnswalg.h:279-282,:1256-1257.
 * Returns ANNB_EFEWRESULTS if any query found fewer than k results (outputs are still filled,
 * missing slots = UINT64_MAX / +inf), mirroring the RuntimeError of the reference. */
ANNB_API int annb_search(annb_index_t *h, const float *queries, const float *tables, int in_space, int64_t B,
                int normalize, int k, int ef, const uint64_t *filter_labels, int filter_space,
                int64_t n_filter, uint64_t *labels_out, float *dists_out, int out_space,
                int64_t *stats_out);

/* Exhaustive ADC over a label subset of the INDEXED nodes (SURVEY.md section 8f rank 4: the brute-force route for
 * very selective filters that HnswIndex.search leaves as a TODO, annlite/core/index/hnsw/index.py:152): the
 * codes of the nodes whose labels are listed are gathered from the graph, scanned with K2 for every query and
 * the k best returned as (labels, dists), ascending (dist, label order of the subset list).  Unknown and
 * deleted labels are skipped; fewer than k candidates -> missing slots = UINT64_MAX / +inf and
 * ANNB_EFEWRESULTS.  Opt-in from the Python side (it changes WHICH results come back compared with the
 * reference's filtered graph walk: these are exact over the subset). */
ANNB_API int annb_scan_subset(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k,
                     const uint64_t *subset_labels, int64_t n_subset, uint64_t *labels_out, float *dists_out);

/* Streaming form of annb_search for serving loops (no stats).  annb_search_submit enqueues upload (host inputs),
 * the walk (tables built inside the kernel) and download (host outputs) of one batch on one of two internal lanes and
 * returns a ticket at once; annb_search_wait blocks until that batch is complete and reports ANNB_EFEWRESULTS like
 * annb_search.  Two batches can be in flight, so the copies of batch i+1 and the under-occupied tail of batch i's
 * launch overlap.  Buffers of a submitted batch (queries, filter labels, outputs) belong to the library until its
 * wait returns; a third submit first waits for the oldest ticket of its lane.  An index with deleted nodes is served
 * by the deletion-aware walk (searchBaseLayerST<true>, hnswalg.h:243-329).
 * annb_search_submit_filtered = knn_query_with_filter (bindings/hnsw_bindings.cpp:393-516) in the same form: the
 * filter label list is uploaded and turned into the by-id bitmap on the batch's own lane; filter_labels == NULL means
 * no filter, a non-NULL list with n_filter == 0 admits nothing.  Queries whose walk outgrew the register lists are
 * re-run on the bitmap walk inside annb_search_wait (annb_fallback_queries counts them) -- or earlier, by the next
 * blocking call on the handle (annb_search, annb_scan_topk, annb_adc_table, annb_add_items, ...): those share device
 * scratch with lane 0 and first settle any such batch, whose ticket stays valid for annb_search_wait. */
ANNB_API int annb_search_submit(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k,
                       int ef, uint64_t *labels_out, float *dists_out, int out_space, int *ticket_out);
ANNB_API int annb_search_submit_filtered(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize,
                                int k, int ef, const uint64_t *filter_labels, int filter_space, int64_t n_filter,
                                uint64_t *labels_out, float *dists_out, int out_space, int *ticket_out);
ANNB_API int annb_search_wait(annb_index_t *h, int ticket);

/* ---- attribute columns and prepared filters ---------------------------------------------------
 * The attribute columns of CellTable (annlite/storage/table.py:160-257), kept by internal id next to the graph:
 * INTEGER -> int64, FLOAT -> double, TEXT -> int32 dictionary code (the code <-> string dictionaries live with the
 * caller).  Every column has a validity bitmap; a row that was never set is NULL.  The host store is the source of
 * truth and follows the graph: it grows with annb_resize_index, new rows are NULL, and annb_init_graph /
 * annb_load_index / annb_set_graph reset every row to NULL (the schema stays).  Its device copy is brought up to
 * date by dirty range on the next annb_filter_prepare.
 *
 * A filter (the WHERE clause CellTable.query runs, annlite/filter.py:17-90) is given as a postfix program of
 * annb_filter_op_t plus a constant pool.  Every leaf pushes one bool per row (NULL rows push false); AND / OR pop two
 * and push one; the program must leave exactly one value.  annb_filter_prepare evaluates it over every row on the
 * GPU, ANDs in "not deleted" and keeps the result as a by-id bitmap owned by the handle.  There is no CPU
 * evaluator: on a host-only handle (device == -1) the store works but prepare and the searches return
 * ANNB_ENODEVICE. */
#define ANNB_ATTR_INTEGER 0 /* int64 values  */
#define ANNB_ATTR_FLOAT 1   /* double values */
#define ANNB_ATTR_TEXT 2    /* int32 dictionary codes (>= 0) */

#define ANNB_MAX_ATTR_COLUMNS 64
#define ANNB_FILTER_MAX_OPS 256
#define ANNB_FILTER_MAX_DEPTH 32
#define ANNB_FILTER_MAX_CONST_BYTES 32768 /* the program and its constants sit in shared memory */

/* op codes.  `a` is a byte offset into the constant pool, `b` a count; numeric constants are 8-byte aligned. */
#define ANNB_FOP_FALSE 0     /* push false                                                            */
#define ANNB_FOP_TRUE 1      /* push true (NULL rows too)                                             */
#define ANNB_FOP_NOTNULL 2   /* push "column col is not NULL"                                         */
#define ANNB_FOP_INT_RANGE 3 /* INTEGER col: lo <= v <= hi, consts[a] = {int64 lo, int64 hi}         */
#define ANNB_FOP_INT_NE 4    /* INTEGER col: v != c, consts[a] = int64 c                              */
#define ANNB_FOP_INT_IN 5    /* INTEGER col: v in consts[a .. a + 8b), int64, sorted ascending         */
#define ANNB_FOP_INT_NIN 6   /* INTEGER col: v not in that list                                       */
#define ANNB_FOP_FLT_RANGE 7 /* FLOAT col: lo <= v <= hi, consts[a] = {double lo, double hi}          */
#define ANNB_FOP_FLT_NE 8    /* FLOAT col: v != c                                                     */
#define ANNB_FOP_FLT_IN 9    /* FLOAT col: v in consts[a .. a + 8b), double, sorted ascending          */
#define ANNB_FOP_FLT_NIN 10  /* FLOAT col: v not in that list                                         */
#define ANNB_FOP_CODE_IN 11  /* TEXT col: bit v of the u32 bitset consts[a ..] of b bits (v >= b: 0)  */
#define ANNB_FOP_AND 12
#define ANNB_FOP_OR 13

typedef struct {
  int32_t op;
  int32_t col;
  int32_t a;
  int32_t b;
} annb_filter_op_t;

/* Declare column `col` (0 <= col < ANNB_MAX_ATTR_COLUMNS, in order) with type ANNB_ATTR_*.  Redeclaring a column
 * with its own type is a no-op; with another type, ANNB_EINVAL. */
ANNB_API int annb_attr_define(annb_index_t *h, int col, int type);
/* Set column `col` of the rows with the given labels: values = n entries of the column's width (int64 / double /
 * int32), valid = n bytes (0 = NULL) or NULL for all valid.  Host memory (space == ANNB_HOST) or device memory.
 * Every label is checked first: an unknown one gives ANNB_ENOTFOUND and nothing is written.  Streamed searches
 * in flight are drained first, as insertions do. */
ANNB_API int annb_attr_set(annb_index_t *h, int col, const uint64_t *labels, int64_t n, const void *values,
                  const uint8_t *valid, int space);
/* Copy column `col` out by internal id (the order of annb_get_labels): values (cap entries of its width) and
 * valid (cap bytes); *n_out = number of rows (the element count).  Either output may be NULL. */
ANNB_API int annb_attr_export(annb_index_t *h, int col, void *values, uint8_t *valid, int64_t cap, int64_t *n_out);
/* Drop every column (schema and values). */
ANNB_API int annb_attr_clear(annb_index_t *h);
/* Validate the program (op codes, columns and their types, constant ranges and alignment, stack balance and depth:
 * ANNB_EINVAL, or ANNB_ELIMIT beyond the limits above) before anything runs, bring the device columns up to date,
 * evaluate it into a bitmap the handle owns and return its id and the number of admitted rows.  One blocking call
 * per filter.  Any later change to the graph, the deletions or the attributes makes the filter stale: using it
 * then returns ANNB_ESTATE (prepare it again). */
ANNB_API int annb_filter_prepare(annb_index_t *h, const annb_filter_op_t *program, int n_ops, const void *consts,
                        int64_t n_const_bytes, int *filter_id, int64_t *count);
/* The labels a prepared filter admits, in internal-id order (insertion order).  Writes min(cap, count) labels
 * and sets *n_out = count. */
ANNB_API int annb_filter_labels(annb_index_t *h, int filter_id, uint64_t *labels_out, int64_t cap, int64_t *n_out);
ANNB_API int annb_filter_release(annb_index_t *h, int filter_id);
/* A prepared filter from a label list (labels, n entries, host or device `space`): the bitmap a search with that list
 * as filter_labels would walk, made once.  Its count is n, as a label list counts (repeats and labels not in the graph
 * included), so annb_search_prepared with it returns what annb_search with the list returns.  It goes stale and is
 * released like a program-prepared filter. */
ANNB_API int annb_filter_prepare_labels(annb_index_t *h, const uint64_t *labels, int64_t n, int space, int *filter_id,
                               int64_t *count);
/* annb_search and annb_search_submit_filtered with a prepared filter in place of the label list: the bitmap is the
 * prepared one and the filter's size is its admitted count; everything else (kernel choice, list sizing, re-runs of
 * overflowing queries, ANNB_EFEWRESULTS) is the filtered route of those calls. */
ANNB_API int annb_search_prepared(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k,
                         int ef, int filter_id, uint64_t *labels_out, float *dists_out, int out_space);
ANNB_API int annb_search_submit_prepared(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize,
                                int k, int ef, int filter_id, uint64_t *labels_out, float *dists_out, int out_space,
                                int *ticket_out);

/* ---- per-query filters ---------------------------------------------------------------------------
 * A serving batch whose requests carry their own filter (the executor's `filter` per request; CellContainer.search
 * runs one CellTable.query per call, annlite/container.py:107-120).  annb_filter_prepare_many evaluates F programs in
 * one pass over the rows: the programs are given back to back (program f = n_ops[f] ops, its pool n_const_bytes[f]
 * bytes, each pool a multiple of 8 and addressed from its own start); a warp runs all of them over its 32 rows.  Sets
 * larger than one launch's shared memory (the two LAUNCH limits) are split into several launches inside the call,
 * which still synchronises once.  Every program is validated as annb_filter_prepare does before anything runs; each
 * referenced column is synced once; each filter gets its own id (annb_filter_release) and goes stale like one from
 * annb_filter_prepare. */
#define ANNB_FILTER_MAX_PER_CALL 1024            /* distinct filters per call (a bitmap is n/8 bytes: 125 KB at 1M rows) */
#define ANNB_FILTER_LAUNCH_MAX_OPS 2048          /* ops one evaluator launch holds in shared memory                       */
#define ANNB_FILTER_LAUNCH_MAX_CONST_BYTES 65536 /* constant bytes one evaluator launch holds                             */
ANNB_API int annb_filter_prepare_many(annb_index_t *h, int F, const annb_filter_op_t *programs, const int *n_ops,
                             const void *consts, const int64_t *n_const_bytes, int *filter_ids_out, int64_t *counts_out);
/* knn_query_with_filter (bindings/hnsw_bindings.cpp:393-516) with one filter per query: query_filter[i] is a prepared
 * filter id, or 0 for no filter (ids start at 1).  Row i is what annb_search_prepared (or annb_search without a filter)
 * returns for query i alone, in ids and distance bits: the batch is split into unfiltered rows, rows whose filter
 * suits hnsw_walk4f and the other filtered rows; each group is one launch over its rows gathered into a contiguous
 * block (hnsw_walk4f's list sized by the group's smallest selectivity), each query reads its own bitmap, queries that
 * outgrew their list are re-run on the bitmap walk with their own bitmap, and the outputs are scattered back.  Any
 * query with fewer than k results gives ANNB_EFEWRESULTS (outputs filled, missing slots UINT64_MAX / +inf).
 * annb_search_submit_multi is the streamed form on the two lanes of annb_search_submit, finished by annb_search_wait
 * (re-runs happen inside the wait). */
ANNB_API int annb_search_multi(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                      const int *query_filter, uint64_t *labels_out, float *dists_out, int out_space);
ANNB_API int annb_search_submit_multi(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k,
                             int ef, const int *query_filter, uint64_t *labels_out, float *dists_out, int out_space,
                             int *ticket_out);

/* ---- shard merge (CellContainer.ivf_search merge rule, annlite/container.py:130-138) ---------- */

/* G per-shard result lists (G,B,k) (as all-gathered over NCCL) -> (B,k) global top-k by
 * (dist, label).  All pointers are device pointers on the handle's GPU. */
ANNB_API int annb_merge_topk(annb_index_t *h, const uint64_t *labels_gbk, const float *dists_gbk, int G,
                    int64_t B, int k, uint64_t *labels_out, float *dists_out);

/* The sharded step without a host synchronisation (annlite/container.py:88-144 spread over G GPUs): a rank's
 * walk (annb_search_submit with DEVICE outputs) writes its (B,k) fp32 distances and (B,k) u64 labels into ONE
 * packed buffer ([dists | pad to 8][labels], rank_stride_bytes long), ONE all-gather of that buffer over NCCL is
 * enqueued on the same lane's stream (annb_lane_stream(ticket & 1) -> torch.cuda.ExternalStream), and
 * annb_merge_topk_packed enqueues the merge of the G gathered buffers on that stream again.  annb_search_wait
 * (ticket) then covers walk + gather + merge.  `lane` = ticket & 1. */
ANNB_API int annb_merge_topk_packed(annb_index_t *h, const void *packed_gathered, int G, int64_t B, int k,
                           int64_t rank_stride_bytes, int64_t labels_offset_bytes, uint64_t *labels_out,
                           float *dists_out, int lane);
ANNB_API int annb_lane_stream(annb_index_t *h, int lane, uint64_t *stream_out);

/* ---- cell sets: multi-cell (IVF) search ---------------------------------------------------------
 * CellContainer.ivf_search (annlite/container.py:88-144) over n_cells existing handles, one HNSW graph per cell, all
 * sharing one PQ codebook.  annb_cellset_create rejects handles on different devices, with a different metric or PQ
 * geometry, or whose codebooks differ, and more than ANNB_MAX_CELLS cells.  `centroids` = the VQ codebook (n_cells,
 * dim) fp32 host (VQCodec.codebook) or NULL; with it, searches without an explicit order probe cells in the order of
 * AnnLite._cell_selection (annlite/index.py:458-466): annlite.math.cdist for the metric, ascending, ties by cell.  The
 * reference's cdist has no inner-product entry, so an IP cell set with centroids is refused (ANNB_EINVAL).  The cell
 * set borrows the handles: they must outlive it and must not be modified during one of its calls.
 *
 * annb_cellset_search: queries (B, dim) host or device (in_space), normalised `normalize` times for the walk (the
 * probe reads them raw); order = (B, n_probe) int32 cells (in_space) or NULL for the centroid order; every cell's
 * device graph is brought up to date first.  Cell c is searched with k_c = min(limit, its live rows) (skipped when 0)
 * and ef_c = max(ef, k_c).  Without deletions, for M = 8 / 256 u8 codes, one launch builds each query's ADC table once
 * and walks all its probed cells (hnsw_walk4's multi-cell form); otherwise -- or with flags & ANNB_CELLS_GENERIC --
 * one annb_search per probed cell.  Both then run the merge of annb_cellset_merge (EUCLIDEAN distances sqrt'ed first,
 * as HnswIndex.search returns them).  Outputs (B, limit): labels, distances, cell of each result; fewer than `limit`
 * results -> UINT64_MAX / +inf / -1.  part_* (optional, out_space): the by-cell scratch (B, n_cells, limit) labels and
 * raw distances, and (B, n_cells, 3) counters as annb_search's stats_out; cells a query does not probe are empty.
 *
 * annb_cellset_merge: the merge alone over a caller-filled by-cell scratch (in_space): labels / dists (B, n_cells,
 * limit) as the per-cell searches return them (sqrt'ed for EUCLIDEAN), counts (B, n_cells) entries per row (a row also
 * ends at its first UINT64_MAX), order (B, n_probe).  In probe order a cell with no results is skipped, and a cell is
 * dropped when the results so far number >= limit and its nearest distance is greater than the last appended cell's
 * largest (container.py:122-123); the kept lists are concatenated and the `limit` smallest returned by (distance,
 * concatenation position), a stable form of container.py:135. */
#define ANNB_MAX_CELLS 256
#define ANNB_CELLS_GENERIC 1 /* annb_cellset_search flag: take the per-cell route even where the fused walk applies */
typedef struct annb_cellset annb_cellset_t;
ANNB_API int annb_cellset_create(annb_index_t *const *handles, int n_cells, const float *centroids, int metric,
                        annb_cellset_t **out);
ANNB_API int annb_cellset_destroy(annb_cellset_t *cs);
ANNB_API int annb_cellset_search(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int normalize,
                        const int32_t *order, int n_probe, int limit, int ef, int flags, uint64_t *labels_out,
                        float *dists_out, int32_t *cells_out, int out_space, uint64_t *part_labels, float *part_dists,
                        int64_t *part_stats);
/* annb_cellset_search with a filter per cell: filter_ids[c] (host, n_cells entries) = a prepared filter of cell c's
 * handle (annb_filter_prepare*, live and not stale: ANNB_EINVAL / ANNB_ESTATE as annb_search_prepared), 0 = the cell
 * admits nothing.  Cell c is searched with k_c = min(limit, its filter's count, its live rows) (skipped when 0) and
 * ef_c = max(ef, k_c): what annb_search_prepared returns for the cell alone.  Where every cell has M = 8 / 256 u8
 * codes and hnsw_walk4f's geometry for max(ef, limit), one launch builds each query's ADC table once and walks all its
 * probed cells with their bitmaps (hnsw_walk4f's multi-cell form, its traversed-only list sized for the most selective
 * cell it walks); a cell too selective for hnsw_walk4f gets the filtered launch annb_search_prepared would run for it,
 * and (query, cell) pairs that outgrew the list are re-run on the bitmap walk of their cell, all on the device.  A
 * probed walk with fewer than k_c results gives ANNB_EFEWRESULTS.  Other geometries, ef > 128 or ANNB_CELLS_GENERIC
 * take one annb_search_prepared per probed cell (whose ANNB_EFEWRESULTS is returned).  Merge, outputs and parts as
 * annb_cellset_search. */
ANNB_API int annb_cellset_search_prepared(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int normalize,
                                 const int32_t *order, int n_probe, int limit, int ef, int flags, const int *filter_ids,
                                 uint64_t *labels_out, float *dists_out, int32_t *cells_out, int out_space,
                                 uint64_t *part_labels, float *part_dists, int64_t *part_stats);
/* What the last annb_cellset_search_prepared did besides the fused launch: (query, cell) pairs re-run on the bitmap
 * walk, and cells served by their own filtered launch. */
ANNB_API int annb_cellset_last_filtered(annb_cellset_t *cs, int64_t *rerun_pairs, int *handle_cells);
ANNB_API int annb_cellset_merge(annb_cellset_t *cs, const uint64_t *labels, const float *dists, const int32_t *counts,
                       const int32_t *order, int in_space, int64_t B, int n_probe, int limit, uint64_t *labels_out,
                       float *dists_out, int32_t *cells_out, int out_space);
/* The probe order alone: (B, n_probe) int32 cells per query, nearest centroid first. */
ANNB_API int annb_cellset_probe(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int n_probe,
                       int32_t *order_out, int out_space);
/* Device time of the last probe / walk (fused launch, or the per-cell searches) / merge in ms, and the route the last
 * annb_cellset_search took (0 = fused walk, 1 = per-cell searches). */
ANNB_API int annb_cellset_last_ms(annb_cellset_t *cs, float *probe_ms, float *walk_ms, float *merge_ms, int *route);

/* ---- introspection for bench / roofline ------------------------------------------------------ */
/* Device time of the last search / scan / table kernel in milliseconds (CUDA events on the
 * handle's stream) and launch counters since creation. */
ANNB_API int annb_last_kernel_ms(annb_index_t *h, float *table_ms, float *search_ms, float *scan_ms);
ANNB_API int annb_launch_count(annb_index_t *h, int64_t *out);
/* number of filtered/deleted batches that outgrew the single-list walk and were re-run on the bitmap walk */
ANNB_API int annb_fallback_count(annb_index_t *h, int64_t *out);
/* ... and how many queries those re-runs covered: only the queries whose list overflowed are redone (the reference's
 * searchBaseLayerSTWithFilter, hnswalg.h:332-440, has no list to overflow) */
ANNB_API int annb_fallback_queries(annb_index_t *h, int64_t *out);
/* How often the device copy of the graph was re-derived from the host graph in full, and how often only the records
 * a small host insertion rewrote were uploaded (the reference searches the structure it inserts into: hnswalg.h:1108;
 * here insertions happen on the host graph and the walk layout on the device follows). */
ANNB_API int annb_sync_counts(annb_index_t *h, int64_t *full_syncs, int64_t *patches);
/* Tuning / A-B / test switches (none changes results): "chunks" (host-buffer pipeline depth of annb_search, 1 = off),
 * "walk_kernel" (plain search: 0 hnsw_walk4 fused, 2 hnsw_walk4 over K1 tables, 1 round-1 kernels), "flagged_kernel"
 * (filter / deletions: 0 hnsw_walk4f where it applies, 1 hnsw_walk_flagged), "flagged_en" (force hnsw_walk4f's
 * traversed-only list to 32 x value entries), "flagged_epl" (force hnsw_walk_flagged with 32 x value entries),
 * "force_general" (1 = filtered route without a filter, 2 = bitmap walk), "scan_kernel" (K2: 0 query-tiled where it
 * applies, 1 round-1 kernel, 2 tiled even for small inputs, 3 first tiled version), "warps_per_cta", "ctas_per_sm",
 * "gpu_build", "gpu_build_frac", "timing", "ip_raw", "dump_tables", "reset_counters". */
ANNB_API int annb_set_option(annb_index_t *h, const char *name, int64_t value);

#ifdef __cplusplus
}
#endif
#endif /* ANNB_H_ */
