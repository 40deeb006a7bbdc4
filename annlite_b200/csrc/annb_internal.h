// annb_internal.h -- shared declarations of libannlite_b200 (not part of the public ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/annb.h"

// ------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------
void annb_set_error(const char *fmt, ...);
#define ANNB_FAIL(code, ...)     \
  do {                           \
    annb_set_error(__VA_ARGS__); \
    return (code);               \
  } while (0)
#define ANNB_CUDA(expr)                                                                     \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      annb_set_error("CUDA error %s at %s:%d (%s)", cudaGetErrorString(_e), __FILE__, __LINE__, #expr); \
      return ANNB_ECUDA;                                                                    \
    }                                                                                       \
  } while (0)

// ------------------------------------------------------------------------------------------
// Host graph: same memory layout as the reference (hnswalg.h:45-49, :66) so that save/load,
// pickle state and builder parity are byte-for-byte checks.
//   level-0 record: [u16 count][u8 flags(bit0 = deleted)][u8 pad][maxM0 x u32 links]
//                   [M x code][u64 label]
//   upper record  : per level [u16 count][u16 pad][maxM x u32 links]
// ------------------------------------------------------------------------------------------
struct HostGraph {
  // geometry
  int M = 16, maxM = 16, maxM0 = 32, ef_construction = 200;
  double mult = 0.0;
  uint64_t seed = 100;
  size_t code_row_bytes = 0;  // n_subvectors * code_bytes
  size_t size_links_level0 = 0, size_per_elem = 0, offset_data = 0, label_offset = 0;
  size_t size_links_per_elem = 0;
  // state
  int64_t max_elements = 0;
  std::atomic<int64_t> count{0};
  int32_t maxlevel = -1;
  uint32_t enterpoint = 0xFFFFFFFFu;
  int64_t num_deleted = 0;
  uint8_t *level0 = nullptr;             // max_elements * size_per_elem
  std::vector<uint8_t *> upper;          // per element: levels * size_links_per_elem (or null)
  std::vector<int32_t> levels;           // element_levels_
  std::unordered_map<uint64_t, uint32_t> label_lookup;
  bool inited = false;
  std::default_random_engine level_gen;  // hnswalg.h:130

  ~HostGraph();
  void clear();
  int init(int64_t max_elems, int M_, int efc, uint64_t seed_, size_t code_row_bytes_);
  int resize(int64_t new_max);
  uint8_t *rec0(uint32_t id) const { return level0 + (size_t)id * size_per_elem; }
  uint8_t *list_at(uint32_t id, int level) const {
    return level == 0 ? rec0(id) : upper[id] + (size_t)(level - 1) * size_links_per_elem;
  }
  const uint8_t *code(uint32_t id) const { return rec0(id) + offset_data; }
  uint64_t label(uint32_t id) const;
  bool deleted(uint32_t id) const { return rec0(id)[2] & 1; }
  int load_file(const char *path, int64_t max_elements_i, size_t code_row_bytes_);
  // Structural soundness of a graph that came from outside (file, pickle state): every count within its list,
  // every link an existing node that has the level it is linked on, entry point and level bounds.  The
  // reference trusts its input; here a bad link would become an out-of-bounds read on the GPU.
  int validate() const;
  int save_file(const char *path) const;
};

// what a host insertion changed, for patching the device graph instead of re-deriving it (capi.cu: patch_device_graph)
struct BuildTrack {
  std::vector<uint32_t> dirty0;  // level-0 records rewritten (with repeats)
  bool upper_dirty = false;      // an upper-level list, a node level > 0 or the entry point changed
  bool untracked = false;        // an in-place update ran: no tracking, re-derive everything
};

// ------------------------------------------------------------------------------------------
// Device graph ("walk layout"): each node's adjacency is co-located with the PQ codes of its
// neighbours so one hop of the walk is ONE contiguous read (DESIGN.md section 3).
//   level-0 record r0[id]  : [maxM0 x u32 link (0xFFFFFFFF = empty)][pad to 16][maxM0 x code_row]
//                            [pad to 16]                                                  (rec0_bytes)
//   upper record  up[l][r] : [maxM x u32 link = record index at level l][pad to 16][maxM x code_row]
//                            [pad to 8][u32 node id][u32 down = record index at level l-1
//                            (node id if l==1)][pad to 16]                                (recu_bytes)
// ------------------------------------------------------------------------------------------
#define ANNB_MAX_LEVELS 32
struct GraphDev {
  const uint8_t *rec0;     // n * rec0_bytes
  const uint8_t *up;       // all upper levels, level l starts at up_off[l] (bytes)
  const uint64_t *labels;  // n
  const uint32_t *deleted; // bitmap by internal id (n/32 words) or nullptr when none deleted
  uint64_t up_off[ANNB_MAX_LEVELS];
  int64_t n;
  int32_t maxlevel;
  uint32_t ep_node;  // entry node id
  uint32_t ep_rec;   // its record index at level maxlevel (== ep_node when maxlevel == 0)
  int32_t maxM, maxM0;
  int32_t rec0_bytes, recu_bytes;
  int32_t code_off0;   // byte offset of the neighbour codes inside a level-0 record (16-aligned)
  int32_t code_offu;   // same for upper records
  int32_t tail_offu;   // byte offset of {u32 node id, u32 down} inside an upper record (8-aligned)
  int32_t M, Ks, code_bytes, code_row;  // code_row = M*code_bytes
  alignas(16) uint8_t ep_code[128];     // code of the entry node (code_row <= 128 bytes)
};

// Wide code rows (ANNB_NARROW_CODE_ROW < code_row <= ANNB_MAX_CODE_ROW): co-locating maxM0 neighbour codes would make a
// level-0 record maxM0 x code_row bytes (24.6 KB at M = 768), so the GraphDev records hold links only and every node's
// code is stored once in a by-internal-id matrix.  GraphDev then reads:
//   level-0 record r0[id]  : [maxM0 x u32 link = node id][pad to 16]                          (rec0_bytes, code_off0 = 0)
//   upper record  up[l][r] : [maxM x u32 link = record index at level l][pad to 16][maxM x u32 node id of that link]
//                            [pad to 8][u32 node id][u32 down][pad to 16]       (recu_bytes; node ids at code_offu)
// and ep_code is unused.  What hnsw_walk_wide reads besides GraphDev and SearchParams:
struct WideDev {
  const uint8_t *codes;   // n x code_stride, node id -> code row (16-byte aligned rows)
  const float *codebook;  // (M, Ks, ds) fp32, as annb_set_codebook received it
  int64_t code_stride;    // bytes between two code rows
  int32_t dim;
};

struct SearchParams {
  const float *tables;  // (B, M, Ks), or nullptr when the walk builds its tables itself (fused K1, hnsw_walk4)
  const float *queries; // (B, D) device, already normalised where the metric asks for it; nullptr = use `tables`
  const float *cbt;     // transposed codebook [m][j/V][c][V] for the fused build
  int cb_vec;           // V: 4 or 2 floats per codeword load
  int ds;               // subvector length
  int is_ip;            // IP / COSINE table form: bias - <cb, q>
  float bias;           // fp32(1/Ks), or 0 for the raw pq_bind form
  int out_internal;     // hnsw_walk4: write internal node ids instead of labels into out_labels (the GPU builder)
  float *dump_tables;   // debug: (B, M, Ks) device buffer that receives the tables the walk used, or nullptr
  int64_t B;
  int k, ef;
  const uint32_t *filter;  // bitmap by internal id, or nullptr
  float selectivity;       // fraction of nodes that can be admitted (filter / not deleted); sizes the flagged list
  uint64_t *out_labels;    // (B,k)
  float *out_dists;        // (B,k)
  int32_t *out_found;      // (B)
  int64_t *out_stats;      // (B,3) or nullptr
  unsigned int *work_counter;
  const uint32_t *qmap;  // bitmap walk only: work item i -> query row (re-run of a subset; then B = #items), or nullptr
  // general-mode scratch (per warp slot)
  uint32_t *visited;      // slots * visited_words
  int64_t visited_words;
  uint32_t *touched;      // slots * touched_cap
  int touched_cap;
  uint64_t *cand;         // slots * cand_cap  (packed: float bits << 32 | id)
  int cand_cap;
  int32_t *overflow_flag;
  // per-query filters (annb_search_multi): B bitmaps by internal id, one per query row of this launch (the row qmap
  // names, for the bitmap walk), nullptr = "not deleted"; nullptr here = every query uses `filter`
  const uint32_t *const *query_filter;
  // multi-cell walk (hnsw_walk4<M, EPL, true>, annb_cellset_search): the device array of the cells' graphs, each
  // query's probe order (B, n_probe) and each cell's k (0 = skip the cell).  Outputs by cell: row q * n_cells + c of
  // out_found / out_stats, and cell_limit entries of out_labels / out_dists per row
  const GraphDev *cells;
  const int32_t *cell_order;
  const int32_t *cell_k;
  int n_cells, n_probe, cell_limit;
  // filtered multi-cell walk (hnsw_walk4f<8, EP, EN, false, true>, annb_cellset_search_prepared): the device array of
  // the cells' prepared bitmaps by internal id, one per cell
  const uint32_t *const *cell_filter;
  // per-query filtered multi-cell walk (hnsw_walk4f<8, EP, EN, true, true>, annb_cellset_search_multi): each query's
  // slot (B); cell_k and cell_filter are then (slots, n_cells) tables, and a cell_filter entry carries its reading in
  // its low bits (bit 0 = "not deleted", bit 1 = size guard), nullptr here = the forms above
  const int32_t *query_slot;
};

// ------------------------------------------------------------------------------------------
// attribute columns (annb_attr_*) and prepared filters (annb_filter_*)
// ------------------------------------------------------------------------------------------
struct AttrColumn {
  int type = -1;                 // ANNB_ATTR_*, -1 = not declared
  int width = 0;                 // bytes per value: 8 (INTEGER / FLOAT) or 4 (TEXT)
  std::vector<uint8_t> vals;     // rows * width, by internal id (host: the source of truth)
  std::vector<uint32_t> valid;   // validity bitmap by internal id
  int64_t dirty_lo = 0, dirty_hi = 0;  // internal ids [lo, hi) not yet on the device
  uint8_t *d_vals = nullptr;     // device copy
  uint32_t *d_valid = nullptr;
  size_t cap_vals = 0, cap_valid = 0;
  int64_t dev_rows = 0;          // rows the device buffers hold
};

// what filter_eval_kernel reads for one column
struct AttrColDev {
  const void *vals;
  const uint32_t *valid;
  int32_t type;
};

struct PreparedFilter {
  uint32_t *bits = nullptr;  // by-id bitmap, (n+31)/32 + 1 words: the layout of S_FLT_BY_ID
  std::shared_ptr<void> block;  // the allocation `bits` lies in, shared by the filters of one prepare call
  int64_t n = 0;             // rows it covers (gd.n at prepare time)
  int64_t count = 0;         // admitted rows
  uint64_t gen = 0;          // annb_index::state_gen at prepare time
  // a label-prepared filter (annb_filter_prepare_labels): the list's entries that name live rows, as internal ids in
  // the caller's order with repeats kept (what annb_scan_subset scans for that list); nullptr for a program's filter
  const uint32_t *ids = nullptr;
  int64_t n_ids = 0;
};

// One subset of a cell scanned exactly for some of the batch's queries (the multi-subset scan, adc_scan.cu).  The
// subset is a bitmap by internal id, compacted in id order (the order annb_filter_labels lists it), or a list of
// internal ids; its code rows and labels are gathered once into `codes` / `labels`.  Each query row in `queries` gets
// the k best (distance, position in the subset) in its pair's row (q * n_cells + cell) of the by-cell scratch.
// Kind SUBSET_LIVE is a cell's live rows in id order: its deletion bitmap read inverted (`bits`, over n_rows ids), or
// with no deletions (bits == nullptr) every row, scanned in place (codes / labels are the cell's own arrays, nothing is
// gathered).
enum { SUBSET_FILTER = 0, SUBSET_LIVE = 1 };
struct SubsetScan {
  const uint32_t *bits;        // bitmap by internal id, or nullptr
  const uint32_t *ids;         // SUBSET_FILTER with bits == nullptr: internal ids in order
  int64_t nwords;              // bitmap words to compact
  int64_t n_rows;              // SUBSET_LIVE: the cell's rows (ids 0..n_rows-1)
  const uint8_t *cell_codes;   // the cell's (rows, 8) own codes by internal id
  const uint64_t *cell_labels; // the cell's labels by internal id
  uint8_t *codes;              // gathered (n, 8) code rows
  uint64_t *labels;            // gathered labels
  unsigned int *block_offs;    // bitmap: per-block counts, then offsets
  int64_t n;                   // subset rows
  const uint32_t *queries;     // query rows that scan the subset
  int32_t nq, k, cell, kind;
};

// Row chunks of one multi-subset scan launch.  rows == 0: each tile's CTA scans its subset whole.  rows > 0: a tile
// (job, first query) becomes one CTA per chunk of `rows` rows; each writes its queries' K best of the chunk (K = the
// launch's largest k) to a list, and the last of the tile's CTAs to finish merges those lists into the pairs' rows.
struct SubsetChunks {
  int64_t rows;
  int G, K;                    // the most chunks of any subset; entries per list
  float *part_d;               // (tile groups, tile width, G, K)
  uint32_t *part_i;
  unsigned int *done;          // (tile groups) chunk CTAs finished, zeroed before the launch
};

// An enqueued search batch, as its flagged queries (found = -1) are re-run on the bitmap walk (capi.cu: rerun_flagged).
// A batch with one filter per query (annb_search_multi / annb_search_submit_multi) is in its gathered row order: the
// rows of each routing group are contiguous; gathered row i is the caller's row dperm[i].  dperm == nullptr: the rows
// are in the caller's order and the gathered outputs are the caller's.
struct MultiBatch {
  int64_t B = 0;
  int k = 0, ef = 0;
  const float *dq = nullptr;                 // gathered queries, normalised (B, dim)
  const uint32_t *filter = nullptr;          // by-id bitmap of every row (nullptr = none) ...
  float selectivity = 1.f;                   // ... and the fraction of nodes it admits
  const uint32_t *const *dqf = nullptr;      // gathered per-query bitmaps (nullptr = no filter), or nullptr
  const uint32_t *dperm = nullptr;           // (B) caller row of each gathered row, or nullptr
  uint64_t *gl = nullptr;                    // gathered outputs (B, k) / (B, k) / (B)
  float *gd = nullptr;
  int32_t *gfound = nullptr;
  int64_t *gstats = nullptr;                 // (B, 3) counters (annb_search), or nullptr
  uint64_t *dl = nullptr;                    // outputs in the caller's row order, on the device
  float *dd = nullptr;
  uint64_t *host_labels = nullptr;           // host outputs, or nullptr (device outputs)
  float *host_dists = nullptr;
  int64_t *host_stats = nullptr;
  int32_t *hfound = nullptr;                 // pinned copy of gfound
  const float *tables = nullptr;             // K1 tables a re-run reuses, or nullptr: it builds them from dq ...
  int table_slot = 0;                        // ... in this scratch slot
  bool timing = false;                       // a re-run records ev[2] / ev[3] around its launch (annb_last_kernel_ms)
};

// ------------------------------------------------------------------------------------------
// the handle
// ------------------------------------------------------------------------------------------
struct annb_index {
  int device = 0;
  int metric = ANNB_METRIC_L2;
  int dim = 0, M = 0, Ks = 0, ds = 0, code_bytes = 1;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;  // second lane of the chunked host-buffer pipeline (annb_search)
  cudaEvent_t ev[6] = {nullptr};  // [0,1] K1, [2,3] K3, [4,5] K2
  std::mutex mu;

  float *d_codebook = nullptr;
  float *d_codebook_t = nullptr;  // transposed copy [m][j/V][c][V] read by the fused table build (hnsw_walk4)
  int cb_vec = 0;                 // V = 4 (ds % 4 == 0), 2 (ds even) or 0 (no fused build)
  std::vector<float> h_codebook;

  // flat code matrix for K2
  uint8_t *d_codes = nullptr;
  int64_t n_codes = 0;

  // graph
  HostGraph g;
  bool dev_dirty = true;
  bool deleted_dirty = false;
  // small host insertions into a graph whose device copy was current: only the rewritten records are uploaded
  BuildTrack patch;
  bool patch_pending = false;
  int64_t patches = 0, full_syncs = 0;
  GraphDev gd{};
  uint8_t *d_rec0 = nullptr, *d_up = nullptr;
  uint64_t *d_labels = nullptr;
  uint32_t *d_deleted = nullptr;
  size_t cap_rec0 = 0, cap_up = 0, cap_labels = 0, cap_deleted = 0;
  size_t up_bytes = 0;  // bytes of d_up the last upload_upper wrote (annb_device_graph_export)
  // every node's own code (n, code_row) by internal id, for the exact subset scan; built on first use per state_gen
  uint8_t *d_own_codes = nullptr;
  size_t cap_own_codes = 0;
  uint64_t own_codes_gen = 0;
  // wide code rows: the by-id code matrix the walk reads (WideDev::codes), kept with the device graph
  uint8_t *d_wide_codes = nullptr;
  size_t cap_wide_codes = 0;

  // scratch (grown on demand)
  void *d_scratch[40] = {nullptr};
  size_t scratch_cap[40] = {0};
  void *h_pinned[6] = {nullptr};
  size_t pinned_cap[6] = {0};
  // asynchronous submit/wait lanes (annb_search_submit): lane i works on stream i with its own scratch
  struct AsyncLane {
    bool busy = false;
    bool flagged = false;  // a filtered / deletion-aware batch: its flagged queries are re-run at wait time
    MultiBatch batch;      // its buffers stay valid until the lane's next submit
  } lanes[2];
  uint32_t next_ticket = 0;

  uint64_t max_label = 0;          // largest label in the graph (filter bitmap sizing)
  bool labels_identity = true;     // label[i] == i for all nodes
  float last_table_ms = 0, last_search_ms = 0, last_scan_ms = 0;
  int64_t launches = 0;
  int64_t flagged_fallback_queries = 0;  // ... and how many queries those re-runs covered
  int64_t flagged_fallbacks = 0;   // batches re-run on the bitmap walk after a flagged-list overflow
  // options
  int64_t opt_warps_per_cta = 0;   // 0 = auto
  int64_t opt_ctas_per_sm = 0;     // 0 = auto
  int64_t opt_force_general = 0;   // use the general (visited + candidate heap) walk always
  int64_t opt_timing = 1;
  int64_t opt_flagged_epl = 0;     // force hnsw_walk_flagged with this list size (entries/32): testing the overflow fallback
  int64_t opt_flagged_en = 0;      // force hnsw_walk4f's traversed-only list to 32 x this many entries (2 / 4 / 8): testing
  int64_t opt_flagged_kernel = 0;  // filtered / deleted search: 0 = hnsw_walk4f where it applies, 1 = hnsw_walk_flagged (round 1)
  int64_t opt_chunks = 0;          // host-buffer search pipeline depth: 0 = auto, 1 = off
  int64_t opt_ip_raw = 0;          // K1 IP form without the 1/Ks bias: T = 0 - ip (pq_bind compatibility)
  int64_t opt_walk_kernel = 0;     // plain search: 0 = hnsw_walk4 with fused K1 (default), 1 = round-1 kernels (K1 +
                                   // hnsw_walk_fast), 2 = hnsw_walk4 over materialised tables (K1 + TMA staging)
  int64_t opt_scan_kernel = 0;     // K2 scan + top-k: 0 = query-tiled kernel where it applies, 1 = round-1 kernel, 2 = tiled even for small inputs (tests), 3 = first tiled version, forced
  int64_t opt_subset_chunk_rows = 0;  // multi-subset scan: 0 = chunked by its size rule, -1 = never, > 0 = chunks of this many rows
  int64_t opt_gpu_build = 1;       // add_items with num_threads != 1 and >= 16384 fresh rows: level-0 insertion on the GPU
  int64_t opt_gpu_build_frac = 16; // a GPU-built batch is at most 1/frac of the graph it is inserted into
  int64_t reserve_nodes = 0;       // sync_device_graph sizes the device graph for this many nodes (GPU builder)
  int64_t opt_dump_tables = 0;     // device pointer: searches copy the tables they used there (debug / parity tests)

  // attribute columns and the filters prepared from them
  std::vector<AttrColumn> attrs;
  std::unordered_map<int, PreparedFilter> filters;
  int next_filter_id = 1;
  uint64_t state_gen = 1;          // bumped by every change to the graph, the deletions or the attributes
};

int annb_scratch(annb_index *h, int slot, size_t bytes, void **out);
int annb_pinned(annb_index *h, int slot, size_t bytes, void **out);

#define ANNB_TRY_RC(expr)    \
  do {                       \
    int _rc = (expr);        \
    if (_rc) return _rc;     \
  } while (0)

// scratch slots (annb_scratch)
enum {
  S_QUERIES = 0, S_TABLES, S_OUT_D, S_OUT_L, S_COUNTER, S_VISITED, S_TOUCHED, S_CAND,
  S_FOUND, S_STATS, S_FLT_LABELS, S_FLT_BY_LABEL, S_FLT_BY_ID, S_RAW0, S_CODES, S_MISC, S_PART_D, S_PART_I,
  S_L1_QUERIES, S_L1_TABLES, S_L1_OUT_D, S_L1_OUT_L, S_L1_FOUND, S_L0_FOUND, S_LANE_COUNTERS, S_QMAP,
  S_L1_FLT_LABELS, S_L1_FLT_BY_LABEL, S_L1_FLT_BY_ID, S_FILTER_PROG, S_FILTER_SCAN, S_FILTER_OUT,
  S_MULTI0, S_MULTI1,  // per-query filter batches of lane 0 (and the blocking call) / lane 1: MultiBatch buffers
  S_SCRATCH_SLOTS
};
static_assert(S_SCRATCH_SLOTS <= 40, "annb_index::d_scratch is too small");

// kernels (launchers)
int launch_l2_normalize(annb_index *h, float *x, int64_t B, int D);
int launch_adc_table(annb_index *h, const float *d_queries, int64_t B, float *d_out);
int launch_scan(annb_index *h, const float *d_table, float *d_out);
int launch_scan_topk(annb_index *h, const float *d_tables, int64_t B, int k, int64_t *d_ids, float *d_dists);
// d_bad_row (or nullptr): set to the first row holding a NaN or an infinity, ~0 if none (reset on h->stream first)
int launch_encode(annb_index *h, const float *d_x, int64_t n, void *d_codes, unsigned long long *d_bad_row);
// ANNB_EINVAL naming the first row of host rows (n, dim) that holds a NaN or an infinity
int check_finite_rows(const float *v, int64_t n, int dim);
#define ANNB_NONFINITE_MSG "array must not contain infs or NaNs"
int launch_pack_rec0(annb_index *h, const uint8_t *d_level0_raw, int64_t n);
int launch_scatter_records(annb_index *h, const uint8_t *d_staged, const uint32_t *d_ids, int64_t cnt, int rec_bytes, uint8_t *d_dst);
// mode: 0 = fast walk (no filter, no deletions), 1 = filtered/deleted walk, kernel chosen automatically
// (flagged single-list walk when its list fits, else the bitmap walk), 2 = bitmap walk
int launch_search(annb_index *h, const SearchParams &p, int mode);
// The route launch_search takes for rows with a filter (filtered) or without, at ef, whose lists are sized by
// `selectivity` (search_selectivity): returns the mode -- 0 = no filter and no deletions, 1, or 2 under
// opt_force_general == 2 -- with *fuse = the walk builds its own tables from the queries (no K1 launch, no (B, M, Ks)
// buffer) and *walk4f = the rows take mode 1 on hnsw_walk4f (either pointer may be null)
int search_route(const annb_index *h, int ef, bool filtered, double selectivity, bool *fuse, bool *walk4f);
// the fraction of the nodes a search can admit: a filter's `count` rows, or (not filtered) the rows not deleted
double search_selectivity(const annb_index *h, bool filtered, int64_t count);
// the work counter of a walk launch and the overflow flag behind it (p.work_counter, or scratch slot 4 when the caller
// passes none; a caller running several launches concurrently passes its own), zeroed on h->stream
int walk_counter(annb_index *h, SearchParams &p);
// f(std::integral_constant<int, EPL>) for the narrowest register list that holds ef entries (32 x EPL, EPL = 2 .. 16)
template <typename F>
int with_epl(int ef, F f) {
  const int epl = (ef + 31) / 32;
  if (epl <= 2) return f(std::integral_constant<int, 2>());
  if (epl <= 4) return f(std::integral_constant<int, 4>());
  if (epl <= 8) return f(std::integral_constant<int, 8>());
  if (epl <= 16) return f(std::integral_constant<int, 16>());
  ANNB_FAIL(ANNB_ELIMIT, "ef=%d exceeds ANNB_MAX_EF=%d", ef, ANNB_MAX_EF);
}
// code rows wider than ANNB_NARROW_CODE_ROW: links-only device records, the by-id code matrix and hnsw_walk_wide
inline bool wide_rows(const annb_index *h) { return (size_t)h->M * h->code_bytes > ANNB_NARROW_CODE_ROW; }
inline int64_t wide_code_stride(const annb_index *h) { return ((int64_t)h->M * h->code_bytes + 15) / 16 * 16; }
// hnsw_walk_wide (walk_wide.cu): every search mode of launch_search for a wide index; distances from p.queries and the
// codebook (p.tables == nullptr) or from p.tables
int launch_walk_wide(annb_index *h, const SearchParams &p);
// hnsw_walk4 (walk_fused.cu): the plain search with the table built inside the walk; returns 1 = not applicable
bool walk4_applicable(const annb_index *h);
bool walk4_can_fuse(const annb_index *h);
int launch_walk4(annb_index *h, const SearchParams &p);
int launch_walk4_cells(annb_index *h, const SearchParams &p);
// hnsw_walk4f (walk_flagged4.cu): the filtered / deletion-aware search on two register lists, same table handling as
// hnsw_walk4; returns 1 = not applicable (then hnsw_walk_flagged or the bitmap walk serve the call)
bool walk4f_applicable(const annb_index *h, int ef, double selectivity);
// ... and its list geometry for that search: (ep, en) = entries per lane of P and N; false = not applicable
bool walk4f_geometry(const annb_index *h, int ef, double selectivity, int *ep_out, int *en_out);
// N's entries per lane as instantiated beside P's ep: the smallest geometry with at least en (en > 0)
int walk4f_round_en(int ep, int en);
int launch_walk4f(annb_index *h, const SearchParams &p);
// the filtered multi-cell walk with lists of (ep, en) entries per lane; returns 1 = not instantiated for these
int launch_walk4f_cells(annb_index *h, const SearchParams &p, int ep, int en);
// capi.cu: a live prepared filter of the handle (ANNB_EINVAL unknown, ANNB_ESTATE stale; the caller holds the lock),
// and annb_search_prepared with annb_search's (B, 3) counters (takes the lock)
int find_prepared_filter(annb_index *h, int filter_id, PreparedFilter **out);
int search_prepared_stats(annb_index *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef, int filter_id,
                          uint64_t *labels_out, float *dists_out, int out_space, int64_t *stats_out);
// the handle's own-code array (annb_index::d_own_codes), current for the graph as it is now (caller holds the lock)
int sync_own_codes(annb_index *h, const uint8_t **out);
// the multi-subset exact scan (adc_scan.cu) over J jobs (d_jobs on the device, `jobs` its host copy): gather every
// subset's rows, then score every job's queries against its subset with the batch's K1 tables (B, 8, 256), k <= 512,
// results straight into the by-cell scratch (found = k, counters {0, 0, n}); M = 8 one-byte codes, Ks = 256 only
bool subset_scan_applicable(const annb_index *h);
int subset_scan_tile_width(int kmax);
// rows per chunk of a launch whose unchunked form has `tiles` CTAs and whose longest subset has `longest` rows (0 =
// unchunked); tiles are int4 {job, first query, chunk, tile group}
int64_t subset_scan_chunk_rows(const annb_index *h, int64_t tiles, int64_t longest);
int launch_subset_scan(annb_index *h, cudaStream_t st, const SubsetScan *d_jobs, const std::vector<SubsetScan> &jobs,
                       const int4 *d_tiles, int64_t n_tiles, const SubsetChunks &ch, const float *tables, int n_cells, int limit,
                       uint64_t *sl, float *sd, int32_t *sfound, int64_t *sstats);
// G ascending (dist, label) lists of k per query -> global k best; *_gstride = distance between two shards' arrays in elements
int launch_merge_topk(annb_index *h, const uint64_t *labels, const float *dists, int G, int64_t B, int k, int64_t l_gstride,
                      int64_t d_gstride, uint64_t *labels_out, float *dists_out, cudaStream_t stream);
int launch_filter_bitmap(annb_index *h, const uint64_t *d_filter_labels, int64_t n_filter, uint32_t *d_by_label,
                         uint32_t *d_by_id);
// attr_filter.cu: evaluate a validated program over rows [0, n) into a by-id bitmap ((n+31)/32 + 1 words) and its
// admitted count (device u64, accumulated: the caller zeroes it); compact a bitmap, less the rows set in d_drop
// (nullable), into the labels of its rows
int launch_filter_eval(annb_index *h, const annb_filter_op_t *d_prog, int n_ops, const void *d_consts, int n_const_bytes,
                       const AttrColDev *cols, int n_cols, int64_t n, const uint32_t *d_deleted, uint32_t *d_bits,
                       unsigned long long *d_count);
// in two steps: launch_filter_count leaves each block's offset in d_block_scratch and the total after them;
// launch_filter_compact then writes that many labels to d_out
int launch_filter_count(annb_index *h, const uint32_t *d_bits, const uint32_t *d_drop, int64_t n, unsigned int *d_block_scratch);
int launch_filter_compact(annb_index *h, const uint32_t *d_bits, const uint32_t *d_drop, int64_t n, const uint64_t *d_labels,
                          uint64_t *d_out, const unsigned int *d_block_scratch);
// blocks the compaction uses for n rows (its scratch holds one u32 per block, plus the total)
int64_t filter_compact_blocks(int64_t n);
// F validated programs in one pass (filter_eval_kernel<true>): program f = ops [d_offs[f], d_offs[f + 1]) of d_prog,
// constant offsets rebased into the one pool; bitmap f at d_bits + f * stride_words, its count added to d_counts[f]
int launch_filter_eval_many(annb_index *h, int F, const annb_filter_op_t *d_prog, const int *d_offs, int n_ops,
                            const void *d_consts, int n_const_bytes, const AttrColDev *cols, int n_cols, int64_t n,
                            const uint32_t *d_deleted, uint32_t *d_bits, int64_t stride_words,
                            unsigned long long *d_counts);
// rows of `row_words` u32: gather (dst[i] = src[idx[i]]) or scatter (dst[idx[i]] = src[i]) for i < n
int launch_rows_copy(annb_index *h, const void *src, void *dst, const uint32_t *d_idx, int64_t n, int row_words, bool scatter);

// host builder
int hnsw_insert_rows(annb_index *h, const uint8_t *codes, const uint64_t *labels, int64_t n, int num_threads,
                     const float *(*table_chunk)(void *, int64_t, int64_t), void *ctx, int64_t chunk_rows,
                     const int32_t *forced_levels = nullptr, BuildTrack *track = nullptr);
// the next n levels the index's generator would hand out (getRandomLevel, hnswalg.h:151-155), in order
int hnsw_draw_levels(annb_index *h, int64_t n, int32_t *out);
// annb_add_items without the handle lock (host insertion; levels forced when given)
int hnsw_host_add(annb_index *h, const float *vectors, const void *codes, const uint64_t *labels, int64_t n, int num_threads,
                  const int32_t *forced_levels);
// level-0 insertion on the GPU (gpu_build.cu); 1 = not applicable, take the host path
int gpu_build_run(annb_index *h, const float *vectors, const uint64_t *labels, int64_t n, int num_threads);
// ... the handle-side part of its rule (geometry, codebook copy, no deletions)
bool gpu_build_geometry(const annb_index *h);
// One cell's share of a cell-set insertion that gpu_build_run would build on the GPU (annb_cellset_add_items)
struct CellBuildJob {
  annb_index *h = nullptr;
  int cell = 0;                   // its index in the cell set (error messages)
  const float *vectors = nullptr; // every row of the call (n, dim)
  std::vector<int64_t> rows;      // the cell's rows of the call, in order
  std::vector<uint64_t> labels;   // their labels
};
struct CellBuildStats {
  double phase1_ms = 0, phase2_ms = 0;
  int64_t rounds = 0;
};
// gpu_build_run for every job at once: phase 1 on a host thread per cell, phase 2 in rounds of every cell's next batch
// on drv's stream (M = 8 codes shared by all cells); each graph comes out as gpu_build_run makes it alone
int gpu_build_cells(annb_index *drv, std::vector<CellBuildJob> &jobs, int num_threads, CellBuildStats *stats);
// capi.cu: what annb_add_items(h, vectors, NULL, labels, n, num_threads) refuses up front (*gpu = it takes the GPU
// builder), and its steps before inserting; the caller holds the handle lock
int add_items_check(annb_index *h, const uint64_t *labels, int64_t n, int num_threads, bool *gpu);
int add_items_enter(annb_index *h);
int sync_device_graph(annb_index *h);
