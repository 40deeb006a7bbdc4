// annb_internal.h -- shared declarations of libannlite_b200 (not part of the public ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <random>
#include <string>
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
};

// a batch with one filter per query (annb_search_multi / annb_search_submit_multi), in its gathered row order: the
// rows of each routing group are contiguous; gathered row i is the caller's row perm[i]
struct MultiBatch {
  int64_t B = 0;
  int k = 0, ef = 0;
  const float *dq = nullptr;                 // gathered queries, normalised (B, dim)
  const uint32_t *const *dqf = nullptr;      // gathered per-query bitmaps (nullptr = no filter)
  const uint32_t *dperm = nullptr;           // (B) caller row of each gathered row
  uint64_t *gl = nullptr;                    // gathered outputs (B, k) / (B, k) / (B)
  float *gd = nullptr;
  int32_t *gfound = nullptr;
  uint64_t *dl = nullptr;                    // outputs in the caller's row order, on the device
  float *dd = nullptr;
  uint64_t *host_labels = nullptr;           // host outputs, or nullptr (device outputs)
  float *host_dists = nullptr;
  int32_t *hfound = nullptr;                 // pinned copy of gfound
  int table_slot = 0;                        // scratch slot of the K1 tables a re-run builds
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

  // scratch (grown on demand)
  void *d_scratch[40] = {nullptr};
  size_t scratch_cap[40] = {0};
  void *h_pinned[6] = {nullptr};
  size_t pinned_cap[6] = {0};
  // asynchronous submit/wait lanes (annb_search_submit): lane i works on stream i with its own scratch
  struct AsyncLane {
    bool busy = false;
    int64_t B = 0;
    int k = 0;
    int32_t *hfound = nullptr;
    // what a filtered / deletion-aware batch needs to re-run its flagged queries at wait time
    bool flagged = false;
    int ef = 0;
    const float *dq = nullptr;          // device queries (normalised), valid until the lane's next submit
    const uint32_t *dfilter = nullptr;  // by-id filter bitmap or nullptr
    float selectivity = 1.f;
    uint64_t *dl = nullptr;
    float *dd = nullptr;
    int32_t *dfound = nullptr;
    uint64_t *host_labels = nullptr;    // host outputs to refresh after a re-run, or nullptr (device outputs)
    float *host_dists = nullptr;
    bool multi = false;                 // a per-query filter batch (annb_search_submit_multi): its state is `mb`
    MultiBatch mb;
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
int launch_encode(annb_index *h, const float *d_x, int64_t n, void *d_codes);
int launch_pack_rec0(annb_index *h, const uint8_t *d_level0_raw, int64_t n);
int launch_scatter_records(annb_index *h, const uint8_t *d_staged, const uint32_t *d_ids, int64_t cnt, int rec_bytes, uint8_t *d_dst);
// mode: 0 = fast walk (no filter, no deletions), 1 = filtered/deleted walk, kernel chosen automatically
// (flagged single-list walk when its list fits, else the bitmap walk), 2 = bitmap walk
int launch_search(annb_index *h, const SearchParams &p, int mode);
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
int launch_walk4f(annb_index *h, const SearchParams &p);
// the filtered multi-cell walk with lists of (ep, en) entries per lane; returns 1 = not instantiated for these
int launch_walk4f_cells(annb_index *h, const SearchParams &p, int ep, int en);
// capi.cu: a live prepared filter of the handle (ANNB_EINVAL unknown, ANNB_ESTATE stale; the caller holds the lock),
// and annb_search_prepared with annb_search's (B, 3) counters (takes the lock)
int find_prepared_filter(annb_index *h, int filter_id, PreparedFilter **out);
int search_prepared_stats(annb_index *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef, int filter_id,
                          uint64_t *labels_out, float *dists_out, int out_space, int64_t *stats_out);
// G ascending (dist, label) lists of k per query -> global k best; *_gstride = distance between two shards' arrays in elements
int launch_merge_topk(annb_index *h, const uint64_t *labels, const float *dists, int G, int64_t B, int k, int64_t l_gstride,
                      int64_t d_gstride, uint64_t *labels_out, float *dists_out, cudaStream_t stream);
int launch_filter_bitmap(annb_index *h, const uint64_t *d_filter_labels, int64_t n_filter, uint32_t *d_by_label,
                         uint32_t *d_by_id);
// attr_filter.cu: evaluate a validated program over rows [0, n) into a by-id bitmap ((n+31)/32 + 1 words) and its
// admitted count (device u64, accumulated: the caller zeroes it); compact a bitmap into the labels of its rows
int launch_filter_eval(annb_index *h, const annb_filter_op_t *d_prog, int n_ops, const void *d_consts, int n_const_bytes,
                       const AttrColDev *cols, int n_cols, int64_t n, const uint32_t *d_deleted, uint32_t *d_bits,
                       unsigned long long *d_count);
int launch_filter_compact(annb_index *h, const uint32_t *d_bits, int64_t n, const uint64_t *d_labels, uint64_t *d_out,
                          unsigned int *d_block_scratch);
// blocks launch_filter_compact uses for n rows (its scratch holds one u32 per block)
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
int sync_device_graph(annb_index *h);
