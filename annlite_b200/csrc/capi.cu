// capi.cu -- the extern "C" boundary of libannlite_b200.so (see include/annb.h).
#include <math_constants.h>
#include <stdarg.h>

#include <algorithm>
#include <limits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <unordered_set>

#include "annb_internal.h"

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
void annb_set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}


int annb_scratch(annb_index *h, int slot, size_t bytes, void **out) {
  if (bytes == 0) bytes = 16;
  if (h->scratch_cap[slot] < bytes) {
    if (h->d_scratch[slot]) {
      ANNB_CUDA(cudaStreamSynchronize(h->stream));
      if (h->stream2) ANNB_CUDA(cudaStreamSynchronize(h->stream2));
      ANNB_CUDA(cudaFree(h->d_scratch[slot]));
      h->d_scratch[slot] = nullptr;
      h->scratch_cap[slot] = 0;
    }
    size_t cap = bytes + bytes / 4;
    cap = (cap + 255) / 256 * 256;
    cudaError_t e = cudaMalloc(&h->d_scratch[slot], cap);
    if (e != cudaSuccess) {
      cudaGetLastError();
      cap = (bytes + 255) / 256 * 256;
      e = cudaMalloc(&h->d_scratch[slot], cap);
    }
    if (e != cudaSuccess) ANNB_FAIL(ANNB_ENOMEM, "cudaMalloc(%zu bytes) failed: %s", cap, cudaGetErrorString(e));
    h->scratch_cap[slot] = cap;
  }
  *out = h->d_scratch[slot];
  return ANNB_OK;
}

int annb_pinned(annb_index *h, int slot, size_t bytes, void **out) {
  if (h->pinned_cap[slot] < bytes) {
    if (h->h_pinned[slot]) {
      ANNB_CUDA(cudaStreamSynchronize(h->stream));
      if (h->stream2) ANNB_CUDA(cudaStreamSynchronize(h->stream2));
      ANNB_CUDA(cudaFreeHost(h->h_pinned[slot]));
      h->h_pinned[slot] = nullptr;
      h->pinned_cap[slot] = 0;
    }
    ANNB_CUDA(cudaMallocHost(&h->h_pinned[slot], bytes));
    h->pinned_cap[slot] = bytes;
  }
  *out = h->h_pinned[slot];
  return ANNB_OK;
}

// Host-only handles (device == -1) exist for the graph container alone -- file I/O, pickle state and
// the host-side insertion algorithm fed with caller-supplied tables.  Every compute entry point
// (tables, scan, encode, search, merge, add_items from vectors) requires a GPU: ANNB_NEED_GPU.
#define ANNB_ENTER(h)                                                        \
  if (!(h)) ANNB_FAIL(ANNB_EINVAL, "null index handle");                     \
  std::lock_guard<std::mutex> _lk((h)->mu);                                  \
  if ((h)->device >= 0) ANNB_CUDA(cudaSetDevice((h)->device))
#define ANNB_NEED_GPU(h) \
  if ((h)->device < 0) ANNB_FAIL(ANNB_ENODEVICE, "this handle is host-only (graph I/O); compute needs a CUDA device: annlite_b200 has no CPU fallback")

#define ANNB_TRY(expr)       \
  do {                       \
    int _rc = (expr);        \
    if (_rc) return _rc;     \
  } while (0)

// ---- attribute rows follow the graph ----------------------------------------------------------------
// size every column to the graph's capacity (new rows are NULL)
static void attr_fit(annb_index *h) {
  const int64_t rows = h->g.inited ? h->g.max_elements : 0;
  for (AttrColumn &c : h->attrs) {
    if (c.type < 0) continue;
    if ((int64_t)c.vals.size() < rows * c.width) c.vals.resize((size_t)rows * c.width, 0);
    if ((int64_t)c.valid.size() < (rows + 31) / 32 + 1) c.valid.resize((size_t)(rows + 31) / 32 + 1, 0u);
  }
}

// the graph was replaced (init / load / adopted state): every row of every column is NULL again, schema kept
static void graph_replaced(annb_index *h) {
  h->state_gen++;
  for (AttrColumn &c : h->attrs) {
    std::fill(c.vals.begin(), c.vals.end(), 0);
    std::fill(c.valid.begin(), c.valid.end(), 0u);
    c.dirty_lo = 0;
    c.dirty_hi = std::numeric_limits<int64_t>::max();
  }
}

// stage an input: returns a device pointer (the caller's own if it already is one)
static int stage_in(annb_index *h, const void *p, int space, size_t bytes, int slot, const void **out) {
  if (space == ANNB_DEVICE) {
    *out = p;
    return ANNB_OK;
  }
  void *d;
  ANNB_TRY(annb_scratch(h, slot, bytes, &d));
  ANNB_CUDA(cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, h->stream));
  *out = d;
  return ANNB_OK;
}

extern "C" {

int annb_version(void) { return ANNB_VERSION; }
const char *annb_last_error(void) { return g_err; }

int annb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int annb_create(int device, int metric, int dim, int n_subvectors, int n_clusters, annb_index_t **out) {
  if (!out) ANNB_FAIL(ANNB_EINVAL, "out is null");
  *out = nullptr;
  if (metric < ANNB_METRIC_L2 || metric > ANNB_METRIC_COSINE) ANNB_FAIL(ANNB_EINVAL, "Space name must be one of l2, ip, or cosine.");
  if (dim <= 0 || n_subvectors <= 0 || n_clusters <= 0) ANNB_FAIL(ANNB_EINVAL, "dim, n_subvectors and n_clusters must be positive");
  if (dim % n_subvectors != 0)
    ANNB_FAIL(ANNB_EINVAL, "Initialization Error, expect HNSW.dim == PQ.n_subvector*PQ.d_subvector, but got:\nHNSW.dim =%d, n_subvectors=%d", dim, n_subvectors);
  if (n_clusters > 65536)
    ANNB_FAIL(ANNB_ELIMIT, "PQ clustering exceed the maximum, annlite set the maximum of clusters = 65536, but got PQ.n_clusters=%d", n_clusters);
  if (device != -1) {
    int ndev = annb_device_count();
    if (ndev <= 0) ANNB_FAIL(ANNB_ENODEVICE, "no CUDA device available: annlite_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) ANNB_FAIL(ANNB_EINVAL, "device %d out of range (have %d)", device, ndev);
    ANNB_CUDA(cudaSetDevice(device));
  }
  annb_index *h = new annb_index();
  h->device = device;
  h->metric = metric;
  h->dim = dim;
  h->M = n_subvectors;
  h->Ks = n_clusters;
  h->ds = dim / n_subvectors;
  h->code_bytes = n_clusters <= 256 ? 1 : 2;
  if ((size_t)h->M * h->code_bytes > ANNB_MAX_CODE_ROW) {
    delete h;
    ANNB_FAIL(ANNB_ELIMIT, "code rows wider than ANNB_MAX_CODE_ROW=%d bytes are not supported (n_subvectors=%d x %d-byte codes)",
              ANNB_MAX_CODE_ROW, n_subvectors, n_clusters <= 256 ? 1 : 2);
  }
  if (device < 0) {
    *out = h;
    return ANNB_OK;
  }
  cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, device);
  cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking);
  for (int i = 0; i < 6 && e == cudaSuccess; i++) e = cudaEventCreate(&h->ev[i]);
  if (e != cudaSuccess) {
    annb_set_error("CUDA error %s while creating stream/events", cudaGetErrorString(e));
    delete h;
    return ANNB_ECUDA;
  }
  *out = h;
  return ANNB_OK;
}

int annb_destroy(annb_index_t *h) {
  if (!h) return ANNB_OK;
  if (h->device < 0) {
    delete h;
    return ANNB_OK;
  }
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (auto &p : h->d_scratch)
    if (p) cudaFree(p);
  for (auto &p : h->h_pinned)
    if (p) cudaFreeHost(p);
  if (h->d_codebook) cudaFree(h->d_codebook);
  if (h->d_codebook_t) cudaFree(h->d_codebook_t);
  if (h->d_codes) cudaFree(h->d_codes);
  if (h->d_rec0) cudaFree(h->d_rec0);
  if (h->d_up) cudaFree(h->d_up);
  if (h->d_labels) cudaFree(h->d_labels);
  if (h->d_deleted) cudaFree(h->d_deleted);
  if (h->d_own_codes) cudaFree(h->d_own_codes);
  if (h->d_wide_codes) cudaFree(h->d_wide_codes);
  for (AttrColumn &c : h->attrs) {
    if (c.d_vals) cudaFree(c.d_vals);
    if (c.d_valid) cudaFree(c.d_valid);
  }
  h->filters.clear();  // the bitmaps live in shared blocks: the last filter of a block frees it
  for (int i = 0; i < 6; i++)
    if (h->ev[i]) cudaEventDestroy(h->ev[i]);
  if (h->stream2) cudaStreamDestroy(h->stream2);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return ANNB_OK;
}

int annb_set_codebook(annb_index_t *h, const float *codebook, int space) {
  ANNB_ENTER(h);
  if (!codebook) ANNB_FAIL(ANNB_EINVAL, "Passed PQ class is none");
  const size_t bytes = (size_t)h->M * h->Ks * h->ds * sizeof(float);
  ANNB_NEED_GPU(h);
  if (!h->d_codebook) ANNB_CUDA(cudaMalloc(&h->d_codebook, bytes));
  ANNB_CUDA(cudaMemcpyAsync(h->d_codebook, codebook, bytes, space == ANNB_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                            h->stream));
  h->h_codebook.resize((size_t)h->M * h->Ks * h->ds);
  if (space == ANNB_DEVICE)
    ANNB_CUDA(cudaMemcpyAsync(h->h_codebook.data(), codebook, bytes, cudaMemcpyDeviceToHost, h->stream));
  else
    memcpy(h->h_codebook.data(), codebook, bytes);
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  // transposed copy for the table build inside the walk (hnsw_walk4): [m][j/V][c][V], V floats per load, so
  // that the 32 lanes of a warp (32 consecutive codewords c) read one contiguous 32*V*4-byte run
  h->cb_vec = (h->ds % 4 == 0) ? 4 : (h->ds % 2 == 0 ? 2 : 0);
  if (h->cb_vec) {
    const int V = h->cb_vec, nv = h->ds / V;
    std::vector<float> t(h->h_codebook.size());
    for (int m = 0; m < h->M; m++)
      for (int c = 0; c < h->Ks; c++)
        for (int j = 0; j < h->ds; j++)
          t[(((size_t)m * nv + j / V) * h->Ks + c) * V + j % V] = h->h_codebook[((size_t)m * h->Ks + c) * h->ds + j];
    if (!h->d_codebook_t) ANNB_CUDA(cudaMalloc(&h->d_codebook_t, bytes));
    ANNB_CUDA(cudaMemcpyAsync(h->d_codebook_t, t.data(), bytes, cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
  }
  return ANNB_OK;
}

int annb_stream(annb_index_t *h, uint64_t *stream_out) {
  if (!h || !stream_out) ANNB_FAIL(ANNB_EINVAL, "null argument");
  *stream_out = (uint64_t)(uintptr_t)h->stream;
  return ANNB_OK;
}

static int lane_wait(annb_index *h, int lane);
static int lane_finish(annb_index *h, int lane, bool check);

// A streamed filtered batch whose walk flagged queries is finished (those queries re-run on the bitmap walk) out of
// the lane's own scratch: queries, filter bitmap, device outputs.  Lane 0 shares these buffers with the blocking entry
// points, so they settle such a batch before they touch them; its ticket stays open for annb_search_wait, which then
// only reports `< k` results.
static int settle_flagged_lanes(annb_index *h) {
  for (int lane = 0; lane < 2; lane++) {
    annb_index::AsyncLane &L = h->lanes[lane];
    if (!L.busy || !L.flagged) continue;
    ANNB_CUDA(cudaStreamSynchronize(lane ? h->stream2 : h->stream));
    ANNB_TRY(lane_finish(h, lane, false));
    L.flagged = false;
  }
  return ANNB_OK;
}

int annb_sync(annb_index_t *h) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  int rc0 = lane_wait(h, 0), rc1 = lane_wait(h, 1);
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream2));
  return rc0 ? rc0 : rc1;
}

// ---- K1 ---------------------------------------------------------------------------------------
// queries (host/device) -> device tables; `d_tables_out` receives the device pointer used.
// queries (host/device) -> device queries, normalised `normalize` times (never the caller's own buffer)
static int stage_queries(annb_index *h, const float *queries, int q_space, int64_t B, int normalize, int slot, const float **dq_out) {
  if (!h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  const size_t qbytes = (size_t)B * h->dim * sizeof(float);
  const float *dq;
  if (normalize > 0 && q_space == ANNB_DEVICE) {  // never modify the caller's buffer
    void *d;
    ANNB_TRY(annb_scratch(h, slot, qbytes, &d));
    ANNB_CUDA(cudaMemcpyAsync(d, queries, qbytes, cudaMemcpyDeviceToDevice, h->stream));
    dq = (const float *)d;
  } else {
    ANNB_TRY(stage_in(h, queries, q_space, qbytes, slot, (const void **)&dq));
  }
  for (int r = 0; r < normalize; r++) ANNB_TRY(launch_l2_normalize(h, const_cast<float *>(dq), B, h->dim));
  *dq_out = dq;
  return ANNB_OK;
}

// queries (host/device) -> device tables (K1 as a kernel of its own: the literal pq_bind calls, K2, insertion)
static int build_tables(annb_index *h, const float *queries, int q_space, int64_t B, int normalize, float *d_tables) {
  const float *dq;
  if (h->opt_timing) cudaEventRecord(h->ev[0], h->stream);
  ANNB_TRY(stage_queries(h, queries, q_space, B, normalize, S_QUERIES, &dq));
  ANNB_TRY(launch_adc_table(h, dq, B, d_tables));
  if (h->opt_timing) cudaEventRecord(h->ev[1], h->stream);
  return ANNB_OK;
}

// Queries whose K1 tables an exhaustive scan builds at once: all B for code rows of <= 128 bytes; for wider rows a
// table is M x Ks x 4 bytes (786 KB at M = 768), so the batch is scanned a chunk at a time within a fixed scratch cap.
static int64_t table_chunk_rows(const annb_index *h, int64_t B) {
  if (!wide_rows(h)) return std::max<int64_t>(B, 1);
  const size_t cap = (size_t)256 << 20, per = (size_t)h->M * h->Ks * sizeof(float);
  return std::max<int64_t>(1, std::min<int64_t>(B, (int64_t)(cap / per)));
}

int annb_adc_table(annb_index_t *h, const float *queries, int q_space, int64_t B, int normalize, float *out, int out_space) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if (B < 0 || (B > 0 && (!queries || !out))) ANNB_FAIL(ANNB_EINVAL, "null queries/out");
  if (B == 0) return ANNB_OK;
  const size_t tbytes = (size_t)B * h->M * h->Ks * sizeof(float);
  float *d_tables = out;
  if (out_space != ANNB_DEVICE) ANNB_TRY(annb_scratch(h, S_TABLES, tbytes, (void **)&d_tables));
  ANNB_TRY(build_tables(h, queries, q_space, B, normalize, d_tables));
  if (out_space != ANNB_DEVICE) {
    ANNB_CUDA(cudaMemcpyAsync(out, d_tables, tbytes, cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
  }
  return ANNB_OK;
}

// ---- K2 ---------------------------------------------------------------------------------------
// A code is an index into a Ks-entry table row.  Where the code type can hold more than Ks (Ks < 256 with u8
// codes, ...) a value from outside -- a caller's array, a file -- is checked once on entry: the kernels and the
// host builder index the table with it unchecked, as the reference does (space_pq.h:30-35).
static int check_code_rows(annb_index *h, const uint8_t *rows, int64_t n, size_t stride) {
  const uint64_t full = h->code_bytes == 1 ? 256ull : (h->code_bytes == 2 ? 65536ull : (1ull << 32));
  if ((uint64_t)h->Ks >= full) return ANNB_OK;
  for (int64_t i = 0; i < n; i++) {
    const uint8_t *r = rows + (size_t)i * stride;
    for (int m = 0; m < h->M; m++) {
      uint32_t v = 0;
      memcpy(&v, r + (size_t)m * h->code_bytes, h->code_bytes);
      if (v >= (uint32_t)h->Ks)
        ANNB_FAIL(ANNB_EINVAL, "PQ code %u (row %lld, subvector %d) is not below n_clusters=%d", v, (long long)i, m, h->Ks);
    }
  }
  return ANNB_OK;
}

int annb_set_codes(annb_index_t *h, const void *codes, int space, int64_t n) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (n < 0 || (n > 0 && !codes)) ANNB_FAIL(ANNB_EINVAL, "null codes");
  if (space != ANNB_DEVICE) ANNB_TRY(check_code_rows(h, (const uint8_t *)codes, n, (size_t)h->M * h->code_bytes));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  if (h->d_codes) {
    ANNB_CUDA(cudaFree(h->d_codes));
    h->d_codes = nullptr;
  }
  h->n_codes = 0;
  if (n == 0) return ANNB_OK;
  const size_t bytes = (size_t)n * h->M * h->code_bytes;
  ANNB_CUDA(cudaMalloc(&h->d_codes, bytes + 16));
  ANNB_CUDA(cudaMemcpyAsync(h->d_codes, codes, bytes, space == ANNB_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                            h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  h->n_codes = n;
  return ANNB_OK;
}

int annb_scan(annb_index_t *h, const float *table, int t_space, float *out_dists, int out_space) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if (!table || !out_dists) ANNB_FAIL(ANNB_EINVAL, "null table/out");
  if (!h->d_codes) ANNB_FAIL(ANNB_ESTATE, "no code matrix: call annb_set_codes first");
  const float *dt;
  ANNB_TRY(stage_in(h, table, t_space, (size_t)h->M * h->Ks * sizeof(float), S_TABLES, (const void **)&dt));
  float *dout = out_dists;
  if (out_space != ANNB_DEVICE) ANNB_TRY(annb_scratch(h, S_OUT_D, (size_t)h->n_codes * sizeof(float), (void **)&dout));
  if (h->opt_timing) cudaEventRecord(h->ev[4], h->stream);
  ANNB_TRY(launch_scan(h, dt, dout));
  if (h->opt_timing) cudaEventRecord(h->ev[5], h->stream);
  if (out_space != ANNB_DEVICE) {
    ANNB_CUDA(cudaMemcpyAsync(out_dists, dout, (size_t)h->n_codes * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
  }
  return ANNB_OK;
}

int annb_scan_topk(annb_index_t *h, const float *queries, const float *tables, int in_space, int64_t B, int k, int64_t *ids,
                   float *dists, int out_space) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if ((queries == nullptr) == (tables == nullptr)) ANNB_FAIL(ANNB_EINVAL, "exactly one of queries / tables must be given");
  if (B < 0 || k <= 0 || !ids || !dists) ANNB_FAIL(ANNB_EINVAL, "bad B/k/outputs");
  if (!h->d_codes) ANNB_FAIL(ANNB_ESTATE, "no code matrix: call annb_set_codes first");
  if (B == 0) return ANNB_OK;
  const size_t TS = (size_t)h->M * h->Ks;
  int64_t *dids = ids;
  float *dd = dists;
  if (out_space != ANNB_DEVICE) {
    ANNB_TRY(annb_scratch(h, S_OUT_L, (size_t)B * k * sizeof(int64_t), (void **)&dids));
    ANNB_TRY(annb_scratch(h, S_OUT_D, (size_t)B * k * sizeof(float), (void **)&dd));
  }
  const int64_t step = table_chunk_rows(h, B);
  for (int64_t b0 = 0; b0 < B; b0 += step) {
    const int64_t nb = std::min(step, B - b0);
    const size_t tbytes = (size_t)nb * TS * sizeof(float);
    const float *dt;
    if (tables) {
      ANNB_TRY(stage_in(h, tables + (size_t)b0 * TS, in_space, tbytes, S_TABLES, (const void **)&dt));
    } else {
      float *t;
      ANNB_TRY(annb_scratch(h, S_TABLES, tbytes, (void **)&t));
      // PQIndex.search builds its table with precompute_adc (L2 form, no normalisation): pq.py:200-224
      ANNB_TRY(build_tables(h, queries + (size_t)b0 * h->dim, in_space, nb, 0, t));
      dt = t;
    }
    if (h->opt_timing && b0 == 0) cudaEventRecord(h->ev[4], h->stream);
    ANNB_TRY(launch_scan_topk(h, dt, nb, k, dids + b0 * k, dd + b0 * k));
  }
  if (h->opt_timing) cudaEventRecord(h->ev[5], h->stream);
  if (out_space != ANNB_DEVICE) {
    ANNB_CUDA(cudaMemcpyAsync(ids, dids, (size_t)B * k * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(dists, dd, (size_t)B * k * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
  }
  return ANNB_OK;
}

// ---- graph ------------------------------------------------------------------------------------
int annb_init_graph(annb_index_t *h, int64_t max_elements, int M, int ef_construction, uint64_t random_seed) {
  ANNB_ENTER(h);
  // M = 1 makes the level multiplier 1/ln(M) infinite (hnswalg.h:47) and the reference's level draw undefined
  if (max_elements < 0 || M < 2 || M > 1024) ANNB_FAIL(ANNB_EINVAL, "bad max_elements / M (2 <= M <= 1024)");
  graph_replaced(h);
  ANNB_TRY(h->g.init(max_elements, M, ef_construction, random_seed, (size_t)h->M * h->code_bytes));
  h->dev_dirty = true;
  return ANNB_OK;
}

int annb_load_index(annb_index_t *h, const char *path, int64_t max_elements) {
  ANNB_ENTER(h);
  if (!path) ANNB_FAIL(ANNB_EINVAL, "null path");
  graph_replaced(h);
  ANNB_TRY(h->g.load_file(path, max_elements, (size_t)h->M * h->code_bytes));
  h->dev_dirty = true;
  if (int rc = check_code_rows(h, h->g.level0 + h->g.offset_data, h->g.count.load(), h->g.size_per_elem)) {
    h->g.clear();
    return rc;
  }
  return ANNB_OK;
}

int annb_save_index(annb_index_t *h, const char *path) {
  ANNB_ENTER(h);
  if (!path) ANNB_FAIL(ANNB_EINVAL, "null path");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  return h->g.save_file(path);
}

int annb_set_graph(annb_index_t *h, const uint8_t *data_level0, uint64_t data_level0_bytes, uint64_t size_data_per_element,
                   uint64_t offset_data, uint64_t label_offset, const uint8_t *link_lists, uint64_t link_lists_bytes,
                   const int32_t *element_levels, int64_t n_element_levels, uint64_t size_links_per_element,
                   int64_t cur_element_count, int64_t max_elements, int32_t max_level, uint32_t enterpoint_node, int max_M,
                   int max_M0, int M, int ef_construction, double mult) {
  ANNB_ENTER(h);
  if (cur_element_count < 0 || cur_element_count > 0xfffffffell || n_element_levels < cur_element_count ||
      (size_data_per_element && data_level0_bytes / size_data_per_element < (uint64_t)cur_element_count) || M < 2 || M > 1024 ||
      ef_construction < 1 || !std::isfinite(mult) || mult < 0.0 || mult > 64.0)
    ANNB_FAIL(ANNB_EINVAL, "graph state is inconsistent with the sizes of its arrays");
  HostGraph &g = h->g;
  const size_t crow = (size_t)h->M * h->code_bytes;
  if (max_elements < cur_element_count) max_elements = cur_element_count;
  graph_replaced(h);
  ANNB_TRY(g.init(max_elements, M, ef_construction, 100, crow));
  if (g.size_per_elem != size_data_per_element) ANNB_FAIL(ANNB_EINVAL, "Invalid value of size_data_per_element_ ");
  if (g.label_offset != label_offset) ANNB_FAIL(ANNB_EINVAL, "Invalid value of label_offset_ ");
  if (g.offset_data != offset_data) ANNB_FAIL(ANNB_EINVAL, "Invalid value of offsetData_ ");
  if (g.maxM != max_M) ANNB_FAIL(ANNB_EINVAL, "Invalid value of maxM_ ");
  if (g.maxM0 != max_M0) ANNB_FAIL(ANNB_EINVAL, "Invalid value of maxM0_ ");
  if (g.size_links_per_elem != size_links_per_element) ANNB_FAIL(ANNB_EINVAL, "Invalid value of size_links_per_element_ ");
  if (cur_element_count < 0 || (cur_element_count > 0 && (!data_level0 || !element_levels))) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  g.mult = mult;
  g.maxlevel = max_level;
  g.enterpoint = enterpoint_node;
  const size_t n = (size_t)cur_element_count;
  if (n) memcpy(g.level0, data_level0, n * g.size_per_elem);
  size_t off = 0;
  for (size_t i = 0; i < n; i++) {
    if (element_levels[i] < 0 || element_levels[i] >= 63 || (element_levels[i] > 0 && !link_lists))
      ANNB_FAIL(ANNB_EINVAL, "Invalid value of element_levels_[%zu]", i);
    g.levels[i] = element_levels[i];
    if (element_levels[i] > 0) {
      const size_t sz = g.size_links_per_elem * (size_t)element_levels[i];
      if (off + sz > link_lists_bytes) {
        for (size_t j = 0; j < i; j++) {
          free(g.upper[j]);
          g.upper[j] = nullptr;
          g.levels[j] = 0;
        }
        g.levels[i] = 0;
        ANNB_FAIL(ANNB_EINVAL, "element_levels_ ask for more link-list bytes than link_lists holds");
      }
      g.upper[i] = (uint8_t *)malloc(sz);
      if (!g.upper[i]) ANNB_FAIL(ANNB_ENOMEM, "Not enough memory: loadIndex failed to allocate linklist");
      memcpy(g.upper[i], link_lists + off, sz);
      off += sz;
    }
  }
  g.count = (int64_t)n;
  g.num_deleted = 0;
  int vrc = g.validate();
  if (vrc == ANNB_OK) vrc = check_code_rows(h, g.level0 + g.offset_data, (int64_t)n, g.size_per_elem);
  if (int rc = vrc) {  // leave an empty, initialised graph behind
    g.count = 0;
    for (size_t i = 0; i < n; i++) {
      free(g.upper[i]);
      g.upper[i] = nullptr;
      g.levels[i] = 0;
    }
    g.maxlevel = -1;
    g.enterpoint = 0xFFFFFFFFu;
    h->dev_dirty = true;
    return rc;
  }
  g.label_lookup.reserve(n);
  for (size_t i = 0; i < n; i++) {
    g.label_lookup[g.label((uint32_t)i)] = (uint32_t)i;
    if (g.deleted((uint32_t)i)) g.num_deleted++;
  }
  h->dev_dirty = true;
  return ANNB_OK;
}

int annb_graph_info(annb_index_t *h, int64_t *cur_element_count, int64_t *max_elements, uint64_t *size_data_per_element,
                    uint64_t *link_lists_bytes, int32_t *max_level, uint32_t *enterpoint_node, int *max_M, int *max_M0, int *M,
                    int *ef_construction, double *mult) {
  ANNB_ENTER(h);
  HostGraph &g = h->g;
  if (!g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  const int64_t n = g.count.load();
  uint64_t lb = 0;
  for (int64_t i = 0; i < n; i++)
    if (g.levels[i] > 0) lb += g.size_links_per_elem * (uint64_t)g.levels[i];
  if (cur_element_count) *cur_element_count = n;
  if (max_elements) *max_elements = g.max_elements;
  if (size_data_per_element) *size_data_per_element = g.size_per_elem;
  if (link_lists_bytes) *link_lists_bytes = lb;
  if (max_level) *max_level = g.maxlevel;
  if (enterpoint_node) *enterpoint_node = g.enterpoint;
  if (max_M) *max_M = g.maxM;
  if (max_M0) *max_M0 = g.maxM0;
  if (M) *M = g.M;
  if (ef_construction) *ef_construction = g.ef_construction;
  if (mult) *mult = g.mult;
  return ANNB_OK;
}

int annb_get_graph(annb_index_t *h, uint8_t *data_level0, uint8_t *link_lists, int32_t *element_levels) {
  ANNB_ENTER(h);
  HostGraph &g = h->g;
  if (!g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  const size_t n = (size_t)g.count.load();
  if (data_level0 && n) memcpy(data_level0, g.level0, n * g.size_per_elem);
  size_t off = 0;
  for (size_t i = 0; i < n; i++) {
    if (element_levels) element_levels[i] = g.levels[i];
    if (g.levels[i] > 0) {
      const size_t sz = g.size_links_per_elem * (size_t)g.levels[i];
      if (link_lists) memcpy(link_lists + off, g.upper[i], sz);
      off += sz;
    }
  }
  return ANNB_OK;
}

int annb_encode(annb_index_t *h, const float *vectors, int v_space, int64_t n, void *codes, int c_space) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if (n < 0 || (n > 0 && (!vectors || !codes))) ANNB_FAIL(ANNB_EINVAL, "null vectors/codes");
  if (!h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  if (n == 0) return ANNB_OK;
  const float *dx;
  ANNB_TRY(stage_in(h, vectors, v_space, (size_t)n * h->dim * sizeof(float), S_QUERIES, (const void **)&dx));
  // codes into scratch, the first non-finite row behind them: the caller's codes are written only for a finite batch
  const size_t cbytes = (size_t)n * h->M * h->code_bytes, flag_at = (cbytes + 7) / 8 * 8;
  uint8_t *dc;
  ANNB_TRY(annb_scratch(h, S_CODES, flag_at + sizeof(unsigned long long), (void **)&dc));
  unsigned long long *d_bad = reinterpret_cast<unsigned long long *>(dc + flag_at), bad = 0;
  ANNB_TRY(launch_encode(h, dx, n, dc, d_bad));
  ANNB_CUDA(cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  if (bad != ~0ull) ANNB_FAIL(ANNB_EINVAL, "row %llu holds a NaN or an infinity: %s", bad, ANNB_NONFINITE_MSG);
  ANNB_CUDA(cudaMemcpyAsync(codes, dc, cbytes, c_space == ANNB_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                            h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  return ANNB_OK;
}

// add_items: tables for each chunk of rows come from K1, double-buffered through pinned memory
struct TableFeed {
  annb_index *h;
  const float *vectors;  // host
  int64_t n, chunk_rows;
  float *pinned[2];
  cudaEvent_t done[2];
  int64_t have_first[2];
  int rc;
};
static int feed_launch(TableFeed *f, int buf, int64_t first) {
  annb_index *h = f->h;
  const int64_t cnt = std::min(f->chunk_rows, f->n - first);
  float *dq, *dt;
  int rc;
  const int qslot = buf ? S_MISC : S_QUERIES, tslot = buf ? S_OUT_D : S_TABLES;
  if ((rc = annb_scratch(h, qslot, (size_t)f->chunk_rows * h->dim * sizeof(float), (void **)&dq))) return rc;
  if ((rc = annb_scratch(h, tslot, (size_t)f->chunk_rows * h->M * h->Ks * sizeof(float), (void **)&dt))) return rc;
  ANNB_CUDA(cudaMemcpyAsync(dq, f->vectors + (size_t)first * h->dim, (size_t)cnt * h->dim * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  // get_dist_mat re-normalises for COSINE (pq.py:309-310) on top of pre_process's pass
  if (h->metric == ANNB_METRIC_COSINE && (rc = launch_l2_normalize(h, dq, cnt, h->dim))) return rc;
  if ((rc = launch_adc_table(h, dq, cnt, dt))) return rc;
  ANNB_CUDA(cudaMemcpyAsync(f->pinned[buf], dt, (size_t)cnt * h->M * h->Ks * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  ANNB_CUDA(cudaEventRecord(f->done[buf], h->stream));
  f->have_first[buf] = first;
  return ANNB_OK;
}
static const float *feed_next(void *ctx, int64_t first, int64_t cnt) {
  TableFeed *f = (TableFeed *)ctx;
  (void)cnt;
  const int buf = (int)((first / f->chunk_rows) & 1);
  if (f->have_first[buf] != first && (f->rc = feed_launch(f, buf, first))) return nullptr;
  if (cudaEventSynchronize(f->done[buf]) != cudaSuccess) {
    annb_set_error("CUDA error while building insertion tables");
    f->rc = ANNB_ECUDA;
    return nullptr;
  }
  const int64_t nxt = first + f->chunk_rows;
  if (nxt < f->n && (f->rc = feed_launch(f, buf ^ 1, nxt))) return nullptr;
  return f->pinned[buf];
}

int annb_add_items(annb_index_t *h, const float *vectors, const void *codes, const uint64_t *labels, int64_t n, int num_threads) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if (n < 0 || (n > 0 && (!vectors || !labels))) ANNB_FAIL(ANNB_EINVAL, "null vectors/labels");
  if (!h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised: call annb_init_graph first");
  if (n == 0) return ANNB_OK;
  ANNB_TRY(check_finite_rows(vectors, n, h->dim));
  h->state_gen++;
  ANNB_CUDA(cudaStreamSynchronize(h->stream));   // insertion reuses search scratch: let streamed searches finish
  ANNB_CUDA(cudaStreamSynchronize(h->stream2));
  // num_threads == 1 is the reference's deterministic single-threaded build; any other value is an unordered
  // concurrent build in the reference too -- large batches of fresh rows then take the GPU builder (deterministic itself)
  if (num_threads != 1 && !codes && h->opt_gpu_build) {
    const int rc = gpu_build_run(h, vectors, labels, n, num_threads);
    if (rc != 1) return rc;
  }
  return hnsw_host_add(h, vectors, codes, labels, n, num_threads, nullptr);
}

}  // extern "C"

// The first row of a host batch (n, dim) holding a NaN or an infinity refuses the batch: a PQ code or a cell cannot be
// chosen for it (scipy.cluster.vq refuses it too).  Insertions check their rows here, before anything is written: the
// GPU builder inserts its first rows on the host before it encodes the rest.
int check_finite_rows(const float *v, int64_t n, int dim) {
  for (int64_t i = 0; i < n; i++) {
    const uint32_t *r = reinterpret_cast<const uint32_t *>(v + (size_t)i * dim);
    uint32_t bad = 0;
    for (int j = 0; j < dim; j++) bad |= (r[j] & 0x7f800000u) == 0x7f800000u;
    if (bad) ANNB_FAIL(ANNB_EINVAL, "row %lld holds a NaN or an infinity: %s", (long long)i, ANNB_NONFINITE_MSG);
  }
  return ANNB_OK;
}

int hnsw_host_add(annb_index *h, const float *vectors, const void *codes, const uint64_t *labels, int64_t n, int num_threads,
                  const int32_t *forced_levels) {
  if (n == 0) return ANNB_OK;
  const size_t crow = (size_t)h->M * h->code_bytes;
  std::vector<uint8_t> own_codes;
  const uint8_t *hc = (const uint8_t *)codes;
  if (hc) ANNB_TRY(check_code_rows(h, hc, n, crow));
  if (!hc) {  // PQCodec.encode on the GPU, chunked
    own_codes.resize((size_t)n * crow);
    const int64_t step = 1 << 18;
    for (int64_t s = 0; s < n; s += step) {
      const int64_t c = std::min(step, n - s);
      float *dx;
      void *dc;
      ANNB_TRY(annb_scratch(h, S_QUERIES, (size_t)c * h->dim * sizeof(float), (void **)&dx));
      ANNB_TRY(annb_scratch(h, S_CODES, (size_t)c * crow, &dc));
      ANNB_CUDA(cudaMemcpyAsync(dx, vectors + (size_t)s * h->dim, (size_t)c * h->dim * sizeof(float), cudaMemcpyHostToDevice, h->stream));
      ANNB_TRY(launch_encode(h, dx, c, dc, nullptr));  // annb_add_items checked the rows
      ANNB_CUDA(cudaMemcpyAsync(own_codes.data() + (size_t)s * crow, dc, (size_t)c * crow, cudaMemcpyDeviceToHost, h->stream));
      ANNB_CUDA(cudaStreamSynchronize(h->stream));
    }
    hc = own_codes.data();
  }
  TableFeed f;
  f.h = h;
  f.vectors = vectors;
  f.n = n;
  const size_t TS = (size_t)h->M * h->Ks;
  // about 64 MB of tables per chunk; wide rows (up to 134 MB per row at M = 512, Ks = 65 536) go down to one row
  const int64_t min_rows = wide_rows(h) ? 1 : 64;
  f.chunk_rows = std::max<int64_t>(min_rows, std::min<int64_t>(8192, (int64_t)((64u << 20) / (TS * sizeof(float)))));
  f.rc = 0;
  for (int b = 0; b < 2; b++) {
    ANNB_TRY(annb_pinned(h, b, (size_t)f.chunk_rows * TS * sizeof(float), (void **)&f.pinned[b]));
    ANNB_CUDA(cudaEventCreateWithFlags(&f.done[b], cudaEventDisableTiming));
    f.have_first[b] = -1;
  }
  // device copy current (possibly with earlier patches pending)?  then remember what this insertion rewrites
  const bool track = !h->dev_dirty && h->d_rec0 && h->gd.n > 0 && !forced_levels;
  BuildTrack tr;
  int rc = hnsw_insert_rows(h, hc, labels, n, num_threads, feed_next, &f, f.chunk_rows, forced_levels, track ? &tr : nullptr);
  cudaStreamSynchronize(h->stream);
  for (int b = 0; b < 2; b++) cudaEventDestroy(f.done[b]);
  if (track && rc == ANNB_OK && !tr.untracked) {
    h->patch.dirty0.insert(h->patch.dirty0.end(), tr.dirty0.begin(), tr.dirty0.end());
    h->patch.upper_dirty |= tr.upper_dirty;
    h->patch_pending = true;
  } else {
    h->dev_dirty = true;
  }
  if (rc == ANNB_ECUDA && f.rc) return f.rc;
  return rc;
}

// What annb_add_items(h, vectors, NULL, labels, n, num_threads) would refuse before it inserts anything (the handle lock
// held); *gpu = it would take the GPU builder (gpu_build_run applies: >= 16384 fresh rows, no stored or repeated labels).
int add_items_check(annb_index *h, const uint64_t *labels, int64_t n, int num_threads, bool *gpu) {
  *gpu = false;
  if (h->device < 0) ANNB_FAIL(ANNB_ENODEVICE, "this handle is host-only (graph I/O); compute needs a CUDA device: annlite_b200 has no CPU fallback");
  if (!h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised: call annb_init_graph first");
  const HostGraph &g = h->g;
  const bool try_gpu = num_threads != 1 && h->opt_gpu_build && n >= 16384 && gpu_build_geometry(h);
  if (try_gpu && g.count.load() + n > g.max_elements) ANNB_FAIL(ANNB_ECAPACITY, "The number of elements exceeds the specified limit");
  int64_t fresh = 0;
  std::unordered_set<uint64_t> seen;
  for (int64_t i = 0; i < n; i++)
    if (g.label_lookup.find(labels[i]) == g.label_lookup.end() && seen.insert(labels[i]).second) fresh++;
  if (g.count.load() + fresh > g.max_elements) ANNB_FAIL(ANNB_ECAPACITY, "The number of elements exceeds the specified limit");
  *gpu = try_gpu && fresh == n;
  return ANNB_OK;
}

// annb_add_items' steps before an insertion (the handle lock held): streamed work settled, the state moved on
int add_items_enter(annb_index *h) {
  ANNB_TRY(settle_flagged_lanes(h));
  h->state_gen++;
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream2));
  return ANNB_OK;
}


extern "C" {

struct HostTables {
  const float *tables;
  size_t TS;
};
static const float *host_tables_next(void *ctx, int64_t first, int64_t) {
  HostTables *t = (HostTables *)ctx;
  return t->tables + (size_t)first * t->TS;
}
int annb_add_items_with_tables(annb_index_t *h, const void *codes, const float *tables, const uint64_t *labels, int64_t n,
                               int num_threads) {
  ANNB_ENTER(h);
  if (n < 0 || (n > 0 && (!codes || !tables || !labels))) ANNB_FAIL(ANNB_EINVAL, "null codes/tables/labels");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised: call annb_init_graph first");
  if (n == 0) return ANNB_OK;
  ANNB_TRY(check_code_rows(h, (const uint8_t *)codes, n, (size_t)h->M * h->code_bytes));
  h->state_gen++;
  HostTables t{tables, (size_t)h->M * h->Ks};
  int rc = hnsw_insert_rows(h, (const uint8_t *)codes, labels, n, num_threads, host_tables_next, &t, n);
  h->dev_dirty = true;
  return rc;
}

int annb_resize_index(annb_index_t *h, int64_t new_max_elements) {
  ANNB_ENTER(h);
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  ANNB_TRY(h->g.resize(new_max_elements));
  h->state_gen++;
  attr_fit(h);
  return ANNB_OK;
}

static int set_deleted(annb_index *h, uint64_t label, bool del) {
  HostGraph &g = h->g;
  auto it = g.label_lookup.find(label);
  if (it == g.label_lookup.end()) ANNB_FAIL(ANNB_ENOTFOUND, "Label not found");
  uint8_t *flags = g.rec0(it->second) + 2;
  if (del) {
    if (*flags & 1) ANNB_FAIL(ANNB_EINVAL, "The requested to delete element is already deleted");
    *flags |= 1;
    g.num_deleted++;
  } else {
    if (!(*flags & 1)) ANNB_FAIL(ANNB_EINVAL, "The requested to undelete element is not deleted");
    *flags &= (uint8_t)~1;
    g.num_deleted--;
  }
  h->deleted_dirty = true;
  h->state_gen++;
  return ANNB_OK;
}
int annb_mark_deleted(annb_index_t *h, uint64_t label) {
  ANNB_ENTER(h);
  return set_deleted(h, label, true);
}
int annb_unmark_deleted(annb_index_t *h, uint64_t label) {
  ANNB_ENTER(h);
  return set_deleted(h, label, false);
}

int annb_element_count(annb_index_t *h, int64_t *out) {
  if (!h || !out) ANNB_FAIL(ANNB_EINVAL, "null argument");
  *out = h->g.inited ? h->g.count.load() : 0;
  return ANNB_OK;
}

int annb_get_labels(annb_index_t *h, uint64_t *labels_out, int64_t cap) {
  ANNB_ENTER(h);
  const int64_t n = std::min<int64_t>(cap, h->g.inited ? h->g.count.load() : 0);
  for (int64_t i = 0; i < n; i++) labels_out[i] = h->g.label((uint32_t)i);
  return ANNB_OK;
}

int annb_get_codes(annb_index_t *h, const uint64_t *labels, int64_t n, void *codes_out) {
  ANNB_ENTER(h);
  HostGraph &g = h->g;
  for (int64_t i = 0; i < n; i++) {
    auto it = g.label_lookup.find(labels[i]);
    if (it == g.label_lookup.end() || g.deleted(it->second)) ANNB_FAIL(ANNB_ENOTFOUND, "Label not found");
    memcpy((uint8_t *)codes_out + (size_t)i * g.code_row_bytes, g.code(it->second), g.code_row_bytes);
  }
  return ANNB_OK;
}

}  // extern "C"

// ---- host graph -> device walk layout ---------------------------------------------------------
static int ensure_dev(void **p, size_t *cap, size_t bytes) {
  if (*cap >= bytes && *p) return ANNB_OK;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  size_t want = bytes + bytes / 8 + 256;
  cudaError_t e = cudaMalloc(p, want);
  if (e != cudaSuccess) {
    cudaGetLastError();
    want = bytes + 256;
    e = cudaMalloc(p, want);
  }
  if (e != cudaSuccess) ANNB_FAIL(ANNB_ENOMEM, "cudaMalloc(%zu bytes) failed: %s", want, cudaGetErrorString(e));
  *cap = want;
  return ANNB_OK;
}

static int upload_deleted(annb_index *h) {
  HostGraph &g = h->g;
  const int64_t n = g.count.load();
  const size_t words = (size_t)(n + 31) / 32 + 1;
  std::vector<uint32_t> bm(words, 0);
  for (int64_t i = 0; i < n; i++)
    if (g.deleted((uint32_t)i)) bm[i >> 5] |= 1u << (i & 31);
  ANNB_TRY(ensure_dev((void **)&h->d_deleted, &h->cap_deleted, words * 4));
  ANNB_CUDA(cudaMemcpyAsync(h->d_deleted, bm.data(), words * 4, cudaMemcpyHostToDevice, h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  h->gd.deleted = h->d_deleted;
  h->deleted_dirty = false;
  return ANNB_OK;
}

// upper levels of the walk layout + entry point, from the host graph (all of it: ~N/16 small records)
static int upload_upper(annb_index *h) {
  HostGraph &g = h->g;
  GraphDev &d = h->gd;
  const int64_t n = g.count.load();
  d.maxlevel = g.maxlevel;
  d.ep_node = g.enterpoint;
  if (g.maxlevel >= ANNB_MAX_LEVELS) ANNB_FAIL(ANNB_ELIMIT, "graph has %d levels (limit %d)", g.maxlevel + 1, ANNB_MAX_LEVELS);
  const bool wide = wide_rows(h);  // upper records carry the links' node ids instead of their codes
  std::vector<uint8_t> up;
  std::vector<uint32_t> map_prev, map_cur;
  size_t off = 0;
  for (int l = 1; l <= g.maxlevel; l++) {
    std::vector<uint32_t> nodes;
    for (int64_t i = 0; i < n; i++)
      if (g.levels[i] >= l) nodes.push_back((uint32_t)i);
    map_cur.assign((size_t)n, 0xffffffffu);
    for (size_t r = 0; r < nodes.size(); r++) map_cur[nodes[r]] = (uint32_t)r;
    d.up_off[l] = off;
    up.resize(off + nodes.size() * (size_t)d.recu_bytes, 0);
    for (size_t r = 0; r < nodes.size(); r++) {
      uint8_t *rec = up.data() + off + r * (size_t)d.recu_bytes;
      const uint32_t u = nodes[r];
      const uint8_t *ll = g.list_at(u, l);
      uint16_t cnt;
      memcpy(&cnt, ll, 2);
      uint32_t *links = reinterpret_cast<uint32_t *>(rec);
      for (int j = 0; j < g.maxM; j++) {
        uint32_t lk = 0xffffffffu;
        if (j < (int)cnt) {
          uint32_t v;
          memcpy(&v, ll + 4 + 4 * j, 4);
          if (map_cur[v] == 0xffffffffu) ANNB_FAIL(ANNB_EINVAL, "Trying to make a link on a non-existent level");
          lk = map_cur[v];
          if (wide) memcpy(rec + d.code_offu + (size_t)j * 4, &v, 4);
          else memcpy(rec + d.code_offu + (size_t)j * d.code_row, g.code(v), (size_t)d.code_row);
        }
        links[j] = lk;
      }
      uint32_t tail[2] = {u, l == 1 ? u : map_prev[u]};
      memcpy(rec + d.tail_offu, tail, 8);
    }
    off += nodes.size() * (size_t)d.recu_bytes;
    if (l == g.maxlevel) d.ep_rec = map_cur[g.enterpoint];
    map_prev.swap(map_cur);
  }
  if (g.maxlevel <= 0) d.ep_rec = g.enterpoint;
  ANNB_TRY(ensure_dev((void **)&h->d_up, &h->cap_up, std::max<size_t>(up.size(), 16)));
  if (!up.empty()) ANNB_CUDA(cudaMemcpyAsync(h->d_up, up.data(), up.size(), cudaMemcpyHostToDevice, h->stream));
  d.up = h->d_up;
  h->up_bytes = up.size();
  if (!wide) memcpy(d.ep_code, g.code(g.enterpoint), (size_t)d.code_row);  // a wide walk reads it from the code matrix
  return ANNB_OK;
}

// A small host insertion into a graph whose device copy was current: upload only what changed -- the rewritten
// level-0 records (packed on the host: links + the neighbours' codes), the new labels, and the upper levels if any
// of them (or the entry point) moved -- instead of re-deriving all N records.
static int patch_device_graph(annb_index *h) {
  HostGraph &g = h->g;
  GraphDev &d = h->gd;
  const int64_t n = g.count.load(), n_old = d.n;
  std::vector<uint32_t> &ids = h->patch.dirty0;
  std::sort(ids.begin(), ids.end());
  ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
  const size_t cnt = ids.size();
  // wide code rows: records hold links only, and the new nodes' rows are appended to the by-id code matrix (the
  // tracked insertion only adds nodes; an in-place update is untracked)
  const bool wide = wide_rows(h);
  const size_t stride = (size_t)wide_code_stride(h);
  if (h->patch.untracked || n < n_old || cnt > (size_t)n / 4 + 64 || (size_t)n * d.rec0_bytes > h->cap_rec0 || (size_t)n * 8 > h->cap_labels ||
      (wide && (size_t)n * stride > h->cap_wide_codes)) {
    h->dev_dirty = true;   // too much changed, or the device buffers are too small: re-derive everything
    return 1;
  }
  uint8_t *hst;
  uint32_t *hid;
  ANNB_TRY(annb_pinned(h, 0, cnt * (size_t)d.rec0_bytes + 16, (void **)&hst));
  ANNB_TRY(annb_pinned(h, 1, cnt * 4 + 16, (void **)&hid));
  for (size_t t = 0; t < cnt; t++) {
    const uint32_t u = ids[t];
    hid[t] = u;
    uint8_t *rec = hst + t * (size_t)d.rec0_bytes;
    memset(rec, 0, (size_t)d.rec0_bytes);
    const uint8_t *ll = g.rec0(u);
    uint16_t c;
    memcpy(&c, ll, 2);
    uint32_t *links = reinterpret_cast<uint32_t *>(rec);
    for (int j = 0; j < g.maxM0; j++) {
      uint32_t lk = 0xffffffffu;
      if (j < (int)c) {
        memcpy(&lk, ll + 4 + 4 * j, 4);
        if (!wide) memcpy(rec + d.code_off0 + (size_t)j * d.code_row, g.code(lk), (size_t)d.code_row);
      }
      links[j] = lk;
    }
  }
  if (wide && n > n_old) {
    std::vector<uint8_t> rows((size_t)(n - n_old) * stride, 0);
    for (int64_t i = n_old; i < n; i++) memcpy(rows.data() + (size_t)(i - n_old) * stride, g.code((uint32_t)i), (size_t)d.code_row);
    ANNB_CUDA(cudaMemcpyAsync(h->d_wide_codes + (size_t)n_old * stride, rows.data(), rows.size(), cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));  // `rows` goes out of scope
  }
  uint8_t *dst;
  uint32_t *did;
  ANNB_TRY(annb_scratch(h, S_RAW0, cnt * (size_t)d.rec0_bytes + 16, (void **)&dst));
  ANNB_TRY(annb_scratch(h, S_QMAP, cnt * 4 + 16, (void **)&did));
  ANNB_CUDA(cudaMemcpyAsync(dst, hst, cnt * (size_t)d.rec0_bytes, cudaMemcpyHostToDevice, h->stream));
  ANNB_CUDA(cudaMemcpyAsync(did, hid, cnt * 4, cudaMemcpyHostToDevice, h->stream));
  ANNB_TRY(launch_scatter_records(h, dst, did, (int64_t)cnt, d.rec0_bytes, h->d_rec0));
  if (n > n_old) {
    std::vector<uint64_t> labels((size_t)(n - n_old));
    for (int64_t i = n_old; i < n; i++) {
      labels[i - n_old] = g.label((uint32_t)i);
      h->max_label = std::max(h->max_label, labels[i - n_old]);
      h->labels_identity &= labels[i - n_old] == (uint64_t)i;
    }
    ANNB_CUDA(cudaMemcpyAsync(h->d_labels + n_old, labels.data(), labels.size() * 8, cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));  // `labels` goes out of scope
  }
  d.n = n;
  if (h->patch.upper_dirty) ANNB_TRY(upload_upper(h));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  ANNB_TRY(upload_deleted(h));
  h->patch_pending = false;
  h->patch = BuildTrack();
  h->patches++;
  return ANNB_OK;
}

int sync_device_graph(annb_index *h) {
  HostGraph &g = h->g;
  if (!g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  if (!h->dev_dirty && !h->deleted_dirty && !h->patch_pending) return ANNB_OK;
  // device buffers are about to be rewritten / reallocated: nothing may still be walking them
  // (streamed searches of annb_search_submit run on both lanes)
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  if (h->stream2) ANNB_CUDA(cudaStreamSynchronize(h->stream2));
  if (!h->dev_dirty && h->patch_pending) {
    const int rc = patch_device_graph(h);
    if (rc != 1) return rc;   // 1 = not patchable: fall through to the full re-derivation
  }
  if (!h->dev_dirty) return upload_deleted(h);
  const int64_t n = g.count.load();
  GraphDev &d = h->gd;
  memset(&d, 0, sizeof(d));
  d.n = n;
  d.M = h->M;
  d.Ks = h->Ks;
  d.code_bytes = h->code_bytes;
  d.code_row = h->M * h->code_bytes;
  d.maxM = g.maxM;
  d.maxM0 = g.maxM0;
  auto up16 = [](size_t v) { return (v + 15) / 16 * 16; };
  const bool wide = wide_rows(h);
  if (wide) {  // links only; upper records carry their links' node ids (annb_internal.h: WideDev)
    d.code_off0 = 0;
    d.rec0_bytes = (int)up16((size_t)4 * g.maxM0);
    d.code_offu = (int)up16((size_t)4 * g.maxM);
    d.tail_offu = (int)(((size_t)d.code_offu + (size_t)g.maxM * 4 + 7) / 8 * 8);
  } else {
    d.code_off0 = (int)up16((size_t)4 * g.maxM0);
    d.rec0_bytes = (int)up16((size_t)d.code_off0 + (size_t)g.maxM0 * d.code_row);
    d.code_offu = (int)up16((size_t)4 * g.maxM);
    d.tail_offu = (int)(((size_t)d.code_offu + (size_t)g.maxM * d.code_row + 7) / 8 * 8);
  }
  d.recu_bytes = (int)up16((size_t)d.tail_offu + 8);
  d.maxlevel = g.maxlevel;
  d.ep_node = g.enterpoint;
  if (n == 0) {
    // an emptied graph (annb_init_graph, or an empty annb_set_graph / annb_load_index): no records, and nothing of the
    // graph it replaced stays behind -- a patch still pending from an insertion into that graph would scatter records of
    // ids this one does not have
    h->max_label = 0;
    h->labels_identity = true;
    h->up_bytes = 0;
    h->patch_pending = false;
    h->patch = BuildTrack();
    h->dev_dirty = false;
    return upload_deleted(h);
  }
  if (g.maxlevel >= ANNB_MAX_LEVELS) ANNB_FAIL(ANNB_ELIMIT, "graph has %d levels (limit %d)", g.maxlevel + 1, ANNB_MAX_LEVELS);

  // level 0: upload the raw records, then gather [links | neighbour codes] on the device
  uint8_t *raw;
  const size_t raw_bytes = (size_t)n * g.size_per_elem;
  ANNB_TRY(annb_scratch(h, S_RAW0, raw_bytes, (void **)&raw));
  ANNB_CUDA(cudaMemcpyAsync(raw, g.level0, raw_bytes, cudaMemcpyHostToDevice, h->stream));
  const int64_t n_alloc = std::max<int64_t>(n, h->reserve_nodes);  // the GPU builder appends nodes in place
  ANNB_TRY(ensure_dev((void **)&h->d_rec0, &h->cap_rec0, (size_t)n_alloc * d.rec0_bytes));
  d.rec0 = h->d_rec0;
  ANNB_TRY(launch_pack_rec0(h, raw, n));
  if (wide) {  // every node's code row, once, from the reference-layout records already on the device
    const size_t stride = (size_t)wide_code_stride(h);
    ANNB_TRY(ensure_dev((void **)&h->d_wide_codes, &h->cap_wide_codes, (size_t)n_alloc * stride));
    ANNB_CUDA(cudaMemcpy2DAsync(h->d_wide_codes, stride, raw + g.offset_data, g.size_per_elem, (size_t)d.code_row, (size_t)n,
                                cudaMemcpyDeviceToDevice, h->stream));
  }

  // labels
  std::vector<uint64_t> labels((size_t)n);
  uint64_t maxl = 0;
  bool ident = true;
  for (int64_t i = 0; i < n; i++) {
    labels[i] = g.label((uint32_t)i);
    maxl = std::max(maxl, labels[i]);
    ident &= labels[i] == (uint64_t)i;
  }
  h->max_label = maxl;
  h->labels_identity = ident;
  ANNB_TRY(ensure_dev((void **)&h->d_labels, &h->cap_labels, (size_t)n_alloc * 8));
  ANNB_CUDA(cudaMemcpyAsync(h->d_labels, labels.data(), (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
  d.labels = h->d_labels;

  ANNB_TRY(upload_upper(h));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  ANNB_TRY(upload_deleted(h));
  h->dev_dirty = false;
  h->patch_pending = false;
  h->patch = BuildTrack();
  h->full_syncs++;
  return ANNB_OK;
}

extern "C" {

// ---- K3 ---------------------------------------------------------------------------------------
// The filter is either a label list (filter_labels, n_filter) or a prepared bitmap (pf, its count standing in for
// n_filter); from there on both take the same route.
static int search_impl(annb_index *h, const float *queries, const float *tables, int in_space, int64_t B, int normalize,
                       int k, int ef, const uint64_t *filter_labels, int filter_space, int64_t n_filter,
                       const PreparedFilter *pf, uint64_t *labels_out, float *dists_out, int out_space, int64_t *stats_out);

int annb_search(annb_index_t *h, const float *queries, const float *tables, int in_space, int64_t B, int normalize, int k,
                int ef, const uint64_t *filter_labels, int filter_space, int64_t n_filter, uint64_t *labels_out,
                float *dists_out, int out_space, int64_t *stats_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  return search_impl(h, queries, tables, in_space, B, normalize, k, ef, filter_labels, filter_space, n_filter, nullptr,
                     labels_out, dists_out, out_space, stats_out);
}

}  // extern "C"

// labels too sparse for a by-label bitmap on the device: labels_to_bitmap resolves them on the host
static bool sparse_labels(const annb_index *h) { return h->max_label > (uint64_t)h->gd.n * 64 + (1ull << 30); }

// labels_to_bitmap's staging buffers in lane `lane`'s scratch: the by-label bitmap and the device copy of host labels
// (*staged = nullptr for device labels; neither for sparse labels)
static int label_staging(annb_index *h, int lane, int filter_space, int64_t n_filter, uint64_t **staged, uint32_t **by_label) {
  *staged = nullptr;
  *by_label = nullptr;
  if (sparse_labels(h)) return ANNB_OK;
  ANNB_TRY(annb_scratch(h, lane ? S_L1_FLT_BY_LABEL : S_FLT_BY_LABEL, ((size_t)(h->max_label >> 5) + 1) * 4, (void **)by_label));
  if (filter_space != ANNB_DEVICE)
    ANNB_TRY(annb_scratch(h, lane ? S_L1_FLT_LABELS : S_FLT_LABELS, (size_t)std::max<int64_t>(n_filter, 1) * 8, (void **)staged));
  return ANNB_OK;
}

// a label list -> the by-id bitmap of the rows it names ((gd.n + 31) / 32 + 1 words), on h->stream, through the
// staging buffers of label_staging
static int labels_to_bitmap(annb_index *h, const uint64_t *filter_labels, int filter_space, int64_t n_filter, uint64_t *staged,
                            uint32_t *by_label, uint32_t *by_id) {
  if (sparse_labels(h)) {
    // resolve the labels through the host's label -> internal id map (the same map mark_deleted uses) and upload the
    // by-id bitmap
    std::vector<uint64_t> tmp;
    const uint64_t *hl = filter_labels;
    if (filter_space == ANNB_DEVICE) {
      tmp.resize((size_t)n_filter);
      ANNB_CUDA(cudaMemcpyAsync(tmp.data(), filter_labels, (size_t)n_filter * 8, cudaMemcpyDeviceToHost, h->stream));
      ANNB_CUDA(cudaStreamSynchronize(h->stream));
      hl = tmp.data();
    }
    std::vector<uint32_t> bm((size_t)(h->gd.n + 31) / 32 + 1, 0u);
    for (int64_t i = 0; i < n_filter; i++) {
      auto it = h->g.label_lookup.find(hl[i]);
      if (it != h->g.label_lookup.end()) bm[it->second >> 5] |= 1u << (it->second & 31);
    }
    ANNB_CUDA(cudaMemcpyAsync(by_id, bm.data(), bm.size() * 4, cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
    return ANNB_OK;
  }
  const uint64_t *dfl = filter_labels;
  if (staged) {
    ANNB_CUDA(cudaMemcpyAsync(staged, filter_labels, (size_t)n_filter * 8, cudaMemcpyHostToDevice, h->stream));
    dfl = staged;
  }
  return launch_filter_bitmap(h, dfl, n_filter, by_label, by_id);
}

// A batch's walk outputs scattered to the caller's rows (dperm), then `found` and the host outputs copied back, on
// h->stream
static int batch_outputs(annb_index *h, const MultiBatch &mb) {
  if (mb.dperm) {
    ANNB_TRY(launch_rows_copy(h, mb.gl, mb.dl, mb.dperm, mb.B, 2 * mb.k, true));
    ANNB_TRY(launch_rows_copy(h, mb.gd, mb.dd, mb.dperm, mb.B, mb.k, true));
  }
  ANNB_CUDA(cudaMemcpyAsync(mb.hfound, mb.gfound, (size_t)mb.B * 4, cudaMemcpyDeviceToHost, h->stream));
  if (mb.host_labels) {
    ANNB_CUDA(cudaMemcpyAsync(mb.host_labels, mb.dl, (size_t)mb.B * mb.k * 8, cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(mb.host_dists, mb.dd, (size_t)mb.B * mb.k * 4, cudaMemcpyDeviceToHost, h->stream));
    if (mb.host_stats) ANNB_CUDA(cudaMemcpyAsync(mb.host_stats, mb.gstats, (size_t)mb.B * 24, cudaMemcpyDeviceToHost, h->stream));
  }
  return ANNB_OK;
}

// A batch's rows in launches: one group for a batch under one filter (or none), three for a batch with one filter per
// query (annb_search_multi): 0 = no filter (the plain walk, or the deletion-aware one), 1 = filters hnsw_walk4f takes
// (its list N sized by the group's smallest selectivity, so one selective filter does not move every query to the
// round-1 kernel), 2 = the other filtered rows (hnsw_walk_flagged / the bitmap walk).  Each group is ONE launch over its
// rows, contiguous in the batch's (gathered) row order.
struct MultiGroup {
  int64_t o = 0, n = 0;  // gathered rows [o, o + n)
  bool filtered = false;
  double s = 1.0;        // the selectivity the group's lists are sized by
  int mode = 0;          // launch_search mode
  bool fuse = false;     // tables built inside the walk (else read from `tables`)
};

// The walk launch of group g of batch mb over the batch's (B, M, Ks) `tables` or, fused, its queries; `dump`: the
// tables it used go to opt_dump_tables, at the group's rows
static SearchParams walk_params(const annb_index *h, const MultiBatch &mb, const MultiGroup &g, const float *tables, bool dump,
                                unsigned int *work_counter) {
  const size_t TS = (size_t)h->M * h->Ks;
  SearchParams p;
  memset(&p, 0, sizeof(p));
  if (g.fuse) {  // hnsw_walk4 / hnsw_walk4f build each query's table in shared memory
    p.queries = mb.dq + g.o * h->dim;
    p.cbt = h->d_codebook_t;
    p.cb_vec = h->cb_vec;
    p.ds = h->ds;
    p.is_ip = h->metric != ANNB_METRIC_L2;
    p.bias = h->opt_ip_raw ? 0.f : (float)(1.0 / (double)h->Ks);
  } else {
    p.tables = tables + g.o * TS;
  }
  if (dump && h->opt_dump_tables) p.dump_tables = reinterpret_cast<float *>(h->opt_dump_tables) + g.o * TS;
  p.B = g.n;
  p.k = mb.k;
  p.ef = mb.ef;
  p.filter = mb.filter;
  p.query_filter = g.filtered && mb.dqf ? mb.dqf + g.o : nullptr;
  p.selectivity = (float)g.s;
  p.out_labels = mb.gl + g.o * mb.k;
  p.out_dists = mb.gd + g.o * mb.k;
  p.out_found = mb.gfound + g.o;
  p.out_stats = mb.gstats ? mb.gstats + g.o * 3 : nullptr;
  p.work_counter = work_counter;
  return p;
}

// The queries of a settled batch that outgrew the flagged walk's list (found = -1, n_over of them) re-run on the bitmap
// walk (exact, any size) through a query-row map, with their own bitmaps, on h->stream: only their rows of the outputs
// are overwritten, then the outputs are copied back again.
static int rerun_flagged(annb_index *h, MultiBatch &mb, int64_t n_over) {
  uint32_t *hmap, *dmap;
  ANNB_TRY(annb_pinned(h, 3, (size_t)n_over * 4, (void **)&hmap));
  ANNB_TRY(annb_scratch(h, S_QMAP, (size_t)n_over * 4, (void **)&dmap));
  const float *tables = mb.tables;
  float *t = nullptr;
  if (!tables) ANNB_TRY(annb_scratch(h, mb.table_slot, (size_t)mb.B * h->M * h->Ks * sizeof(float), (void **)&t));
  int64_t w = 0;
  for (int64_t b = 0; b < mb.B; b++)
    if (mb.hfound[b] < 0) hmap[w++] = (uint32_t)b;
  ANNB_CUDA(cudaMemcpyAsync(dmap, hmap, (size_t)n_over * 4, cudaMemcpyHostToDevice, h->stream));
  if (!tables) {  // the walk built its tables in shared memory: the bitmap walk reads them from HBM (K1, all rows)
    ANNB_TRY(launch_adc_table(h, mb.dq, mb.B, t));
    tables = t;
  }
  MultiGroup g;
  g.n = n_over;
  g.filtered = true;
  g.s = mb.selectivity;
  SearchParams p = walk_params(h, mb, g, tables, false, nullptr);
  p.qmap = dmap;
  if (mb.timing && h->opt_timing) cudaEventRecord(h->ev[2], h->stream);
  ANNB_TRY(launch_search(h, p, 2));
  if (mb.timing && h->opt_timing) cudaEventRecord(h->ev[3], h->stream);
  ANNB_TRY(batch_outputs(h, mb));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  h->flagged_fallbacks++;
  h->flagged_fallback_queries += n_over;
  return ANNB_OK;
}

// A settled batch: its flagged queries re-run (`flagged` = its walks can flag queries), then (check) ANNB_EFEWRESULTS
// where a query has fewer than k results (hnsw_bindings.cpp:342-345)
static int finish_batch(annb_index *h, MultiBatch &mb, bool flagged, bool check) {
  if (flagged) {
    int64_t n_over = 0;
    for (int64_t b = 0; b < mb.B; b++) n_over += mb.hfound[b] < 0;
    if (n_over) ANNB_TRY(rerun_flagged(h, mb, n_over));
  }
  if (check)
    for (int64_t b = 0; b < mb.B; b++)
      if (mb.hfound[b] < mb.k)
        ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  return ANNB_OK;
}

// Enqueue a planned batch on h->stream with the scratch of `lane` (lane 0 also serves the blocking calls): stage and
// normalise the queries -- gathered into the groups' row order when the batch has a row map (gathered row i is the
// caller's row (*perm)[i], with bitmap (*qf)[i]) --, run K1 for the groups whose walk does not build its tables (or
// take the caller's `tables`: one group, not fused), build the label list's bitmap, launch one walk per non-empty group,
// then scatter the outputs back to the caller's rows and copy them out (batch_outputs).  A blocking call uses the
// handle's own found slot, work counter and pinned slot 2; it times K1 (ev[0], ev[1]; a gathered batch times its K1
// with its walks) and its walks (ev[2], ev[3]), dumps its tables (opt_dump_tables) and, in the caller's row order,
// leaves them to a re-run.  *flagged = some walk can flag queries for a re-run.
static int enqueue_batch(annb_index *h, int lane, bool blocking, const float *queries, const float *tables, int in_space, int64_t B,
                         int normalize, int k, int ef_eff, const MultiGroup *grp, int n_grp, const std::vector<uint32_t> *perm,
                         const std::vector<const uint32_t *> *qf, const uint64_t *filter_labels, int filter_space, int64_t n_filter,
                         const uint32_t *filter_bits, uint64_t *labels_out, float *dists_out, int out_space, int64_t *stats_out,
                         MultiBatch &mb, bool *flagged) {
  const bool host_in = in_space != ANNB_DEVICE, host_out = out_space != ANNB_DEVICE, gathered = perm != nullptr;
  const size_t TS = (size_t)h->M * h->Ks, dim = (size_t)h->dim;
  bool need_tables = false;
  *flagged = false;
  for (int i = 0; i < n_grp; i++) {
    need_tables |= grp[i].n && !grp[i].fuse;
    *flagged |= grp[i].n && grp[i].mode == 1;
  }
  mb = MultiBatch();
  mb.B = B;
  mb.k = k;
  mb.ef = ef_eff;
  mb.selectivity = gathered ? 1.f : (float)grp[0].s;
  mb.dl = labels_out;
  mb.dd = dists_out;
  mb.gstats = stats_out;
  mb.table_slot = lane ? S_L1_TABLES : S_TABLES;
  // all scratch first: a (re)allocation synchronises both lanes, which is only safe before enqueuing
  if (host_out) {
    ANNB_TRY(annb_scratch(h, lane ? S_L1_OUT_L : S_OUT_L, (size_t)B * k * 8, (void **)&mb.dl));
    ANNB_TRY(annb_scratch(h, lane ? S_L1_OUT_D : S_OUT_D, (size_t)B * k * 4, (void **)&mb.dd));
    if (stats_out) ANNB_TRY(annb_scratch(h, S_STATS, (size_t)B * 24, (void **)&mb.gstats));
    mb.host_labels = labels_out;
    mb.host_dists = dists_out;
    mb.host_stats = stats_out;
  }
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t o_perm = al((size_t)B * 8), o_found = o_perm + al((size_t)B * 4), o_gl = o_found + al((size_t)B * 4),
               o_gd = o_gl + al((size_t)B * k * 8), o_q = o_gd + al((size_t)B * k * 4), total = o_q + al((size_t)B * dim * 4);
  uint8_t *mq = nullptr;  // a gathered batch: bitmaps, row map, found, outputs and queries, in the gathered order
  if (gathered) {
    ANNB_TRY(annb_scratch(h, lane ? S_MULTI1 : S_MULTI0, total, (void **)&mq));
    mb.dqf = reinterpret_cast<const uint32_t *const *>(mq);
    mb.dperm = reinterpret_cast<const uint32_t *>(mq + o_perm);
    mb.gfound = reinterpret_cast<int32_t *>(mq + o_found);
    mb.gl = reinterpret_cast<uint64_t *>(mq + o_gl);
    mb.gd = reinterpret_cast<float *>(mq + o_gd);
  } else {
    ANNB_TRY(annb_scratch(h, blocking ? S_FOUND : (lane ? S_L1_FOUND : S_L0_FOUND), (size_t)B * 4, (void **)&mb.gfound));
    mb.gl = mb.dl;
    mb.gd = mb.dd;
  }
  float *dq = nullptr, *dtab = const_cast<float *>(tables);  // device queries are read in place unless normalised
  if (queries && (host_in || (normalize > 0 && !gathered)))
    ANNB_TRY(annb_scratch(h, lane ? S_L1_QUERIES : S_QUERIES, (size_t)B * dim * 4, (void **)&dq));
  if (need_tables && (!tables || host_in)) ANNB_TRY(annb_scratch(h, lane ? S_L1_TABLES : S_TABLES, (size_t)B * TS * 4, (void **)&dtab));
  uint32_t *by_id = const_cast<uint32_t *>(filter_bits), *by_label = nullptr;
  uint64_t *staged = nullptr;
  if (filter_labels) {
    ANNB_TRY(annb_scratch(h, lane ? S_L1_FLT_BY_ID : S_FLT_BY_ID, ((size_t)(h->gd.n + 31) / 32 + 1) * 4, (void **)&by_id));
    ANNB_TRY(label_staging(h, lane, filter_space, n_filter, &staged, &by_label));
  }
  mb.filter = by_id;
  unsigned int *counter = nullptr;  // blocking: the handle's own (walk_counter)
  if (!blocking) {
    ANNB_TRY(annb_scratch(h, S_LANE_COUNTERS, 512, (void **)&counter));
    counter += 64 * lane;
  }
  ANNB_TRY(annb_pinned(h, blocking ? 2 : 4 + lane, (size_t)B * 4, (void **)&mb.hfound));

  const bool timing = blocking && h->opt_timing, time_k1 = timing && !gathered && need_tables && !tables;
  if (time_k1) cudaEventRecord(h->ev[0], h->stream);
  if (gathered) {
    std::vector<uint8_t> meta(o_found, 0);
    memcpy(meta.data(), qf->data(), (size_t)B * 8);
    memcpy(meta.data() + o_perm, perm->data(), (size_t)B * 4);
    ANNB_CUDA(cudaMemcpyAsync(mq, meta.data(), o_found, cudaMemcpyHostToDevice, h->stream));
  }
  if (queries) {
    const float *src = queries;
    if (dq) {
      ANNB_CUDA(cudaMemcpyAsync(dq, queries, (size_t)B * dim * 4, host_in ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice,
                                h->stream));
      src = dq;
    }
    if (gathered) {
      ANNB_TRY(launch_rows_copy(h, src, mq + o_q, mb.dperm, B, (int)dim, false));
      src = reinterpret_cast<float *>(mq + o_q);
    }
    for (int r = 0; r < normalize; r++) ANNB_TRY(launch_l2_normalize(h, const_cast<float *>(src), B, (int)dim));
    mb.dq = src;
  } else if (host_in) {
    ANNB_CUDA(cudaMemcpyAsync(dtab, tables, (size_t)B * TS * 4, cudaMemcpyHostToDevice, h->stream));
  }
  if (timing && gathered) cudaEventRecord(h->ev[2], h->stream);
  for (int i = 0; i < n_grp && !tables; i++)
    if (grp[i].n && !grp[i].fuse) ANNB_TRY(launch_adc_table(h, mb.dq + grp[i].o * dim, grp[i].n, dtab + grp[i].o * TS));
  if (time_k1) cudaEventRecord(h->ev[1], h->stream);
  if (filter_labels) ANNB_TRY(labels_to_bitmap(h, filter_labels, filter_space, n_filter, staged, by_label, by_id));
  if (timing && !gathered) cudaEventRecord(h->ev[2], h->stream);
  for (int i = 0; i < n_grp; i++)
    if (grp[i].n) ANNB_TRY(launch_search(h, walk_params(h, mb, grp[i], dtab, blocking && !gathered, counter), grp[i].mode));
  if (timing) cudaEventRecord(h->ev[3], h->stream);
  ANNB_TRY(batch_outputs(h, mb));
  if (blocking && !gathered) {
    mb.tables = need_tables ? dtab : nullptr;
    mb.timing = true;
  }
  return ANNB_OK;
}

// The host-buffer plain search as a pipeline of nch chunks on two streams: H2D of chunk c+1 overlaps the walk of chunk
// c, the walk of chunk c+1 fills the SMs that chunk c's persistent launch leaves idle in its tail, and D2H of chunk c
// overlaps the walk of chunk c+1.
static int search_chunked(annb_index *h, const float *queries, int64_t B, int normalize, int k, int ef_eff, bool fuse, int nch,
                          uint64_t *labels_out, float *dists_out, int64_t *stats_out) {
  const size_t TS = (size_t)h->M * h->Ks;
  MultiBatch mb;
  mb.k = k;
  mb.ef = ef_eff;
  float *dq, *dtab = nullptr;
  unsigned int *counters;
  int32_t *hfound;
  ANNB_TRY(annb_scratch(h, S_OUT_L, (size_t)B * k * 8, (void **)&mb.gl));
  ANNB_TRY(annb_scratch(h, S_OUT_D, (size_t)B * k * 4, (void **)&mb.gd));
  ANNB_TRY(annb_scratch(h, S_FOUND, (size_t)B * 4, (void **)&mb.gfound));
  if (stats_out) ANNB_TRY(annb_scratch(h, S_STATS, (size_t)B * 24, (void **)&mb.gstats));
  ANNB_TRY(annb_scratch(h, S_QUERIES, (size_t)B * h->dim * sizeof(float), (void **)&dq));
  if (!fuse) ANNB_TRY(annb_scratch(h, S_TABLES, (size_t)B * TS * sizeof(float), (void **)&dtab));
  ANNB_TRY(annb_scratch(h, S_COUNTER, 256 * 9, (void **)&counters));
  ANNB_TRY(annb_pinned(h, 2, (size_t)B * 4, (void **)&hfound));
  mb.dq = dq;
  ANNB_CUDA(cudaStreamSynchronize(h->stream));  // scratch (re)allocation and earlier work are settled
  cudaStream_t lanes[2] = {h->stream, h->stream2};
  cudaStream_t saved = h->stream;
  int rc = ANNB_OK;
  for (int c = 0; c < nch && rc == ANNB_OK; c++) {
    MultiGroup g;
    g.o = B * c / nch;
    g.n = B * (c + 1) / nch - g.o;
    g.fuse = fuse;
    const int64_t b0 = g.o, nb = g.n;
    h->stream = lanes[c & 1];
    if (cudaMemcpyAsync(dq + b0 * h->dim, queries + b0 * h->dim, (size_t)nb * h->dim * sizeof(float),
                        cudaMemcpyHostToDevice, h->stream) != cudaSuccess) {
      rc = ANNB_ECUDA;
      break;
    }
    for (int r = 0; r < normalize && rc == ANNB_OK; r++) rc = launch_l2_normalize(h, dq + b0 * h->dim, nb, h->dim);
    if (rc == ANNB_OK && !fuse) rc = launch_adc_table(h, dq + b0 * h->dim, nb, dtab + b0 * TS);
    if (rc != ANNB_OK) break;
    if (c == 0 && h->opt_timing) cudaEventRecord(h->ev[2], h->stream);
    rc = launch_search(h, walk_params(h, mb, g, dtab, true, counters + 64 * (c + 1)), g.mode);
    if (rc != ANNB_OK) break;
    if (c == nch - 1 && h->opt_timing) cudaEventRecord(h->ev[3], h->stream);
    cudaMemcpyAsync(hfound + b0, mb.gfound + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost, h->stream);
    cudaMemcpyAsync(labels_out + b0 * k, mb.gl + b0 * k, (size_t)nb * k * 8, cudaMemcpyDeviceToHost, h->stream);
    cudaMemcpyAsync(dists_out + b0 * k, mb.gd + b0 * k, (size_t)nb * k * 4, cudaMemcpyDeviceToHost, h->stream);
    if (stats_out) cudaMemcpyAsync(stats_out + b0 * 3, mb.gstats + b0 * 3, (size_t)nb * 24, cudaMemcpyDeviceToHost, h->stream);
  }
  h->stream = saved;
  cudaError_t e1 = cudaStreamSynchronize(h->stream), e2 = cudaStreamSynchronize(h->stream2);
  if (rc != ANNB_OK) {
    if (rc == ANNB_ECUDA) annb_set_error("CUDA error in the chunked search pipeline: %s", cudaGetErrorString(cudaGetLastError()));
    return rc;
  }
  if (e1 != cudaSuccess || e2 != cudaSuccess)
    ANNB_FAIL(ANNB_ECUDA, "CUDA error %s in the chunked search pipeline", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
  for (int64_t b = 0; b < B; b++)
    if (hfound[b] < k)
      ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  return ANNB_OK;
}

// the one group of a batch under one filter that admits n_filter rows (filtered), or under none
static MultiGroup single_group(const annb_index *h, int64_t B, int ef_eff, bool filtered, int64_t n_filter) {
  MultiGroup g;
  g.n = B;
  g.filtered = filtered;
  g.s = search_selectivity(h, filtered, n_filter);
  g.mode = search_route(h, ef_eff, filtered, g.s, &g.fuse, nullptr);
  return g;
}

static int search_impl(annb_index *h, const float *queries, const float *tables, int in_space, int64_t B, int normalize,
                       int k, int ef, const uint64_t *filter_labels, int filter_space, int64_t n_filter,
                       const PreparedFilter *pf, uint64_t *labels_out, float *dists_out, int out_space, int64_t *stats_out) {
  const bool has_filter = filter_labels || pf;
  if (pf) n_filter = pf->count;
  ANNB_TRY(settle_flagged_lanes(h));
  if ((queries == nullptr) == (tables == nullptr)) ANNB_FAIL(ANNB_EINVAL, "exactly one of queries / tables must be given");
  if (B < 0 || k <= 0 || ef <= 0 || !labels_out || !dists_out) ANNB_FAIL(ANNB_EINVAL, "bad B/k/ef/outputs");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  ANNB_TRY(sync_device_graph(h));
  if (B == 0) return ANNB_OK;
  const int ef_eff = std::max(ef, k);  // hnswalg.h:1279
  if (ef_eff > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "max(ef, k)=%d exceeds ANNB_MAX_EF=%d", ef_eff, ANNB_MAX_EF);
  if (h->gd.n == 0) {  // empty index: searchKnn returns nothing (hnswalg.h:1240)
    ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  }
  if (queries && !h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  MultiGroup g = single_group(h, B, ef_eff, has_filter, n_filter);
  g.fuse &= !tables;  // the caller's tables: the walk reads them
  int nch = (int)h->opt_chunks;
  if (nch == 0) nch = (B >= 32768) ? 4 : (B >= 4096 ? 2 : 1);
  if (nch > 8) nch = 8;
  if (queries && in_space != ANNB_DEVICE && out_space != ANNB_DEVICE && g.mode == 0 && nch > 1 && B >= 2 * nch)
    return search_chunked(h, queries, B, normalize, k, ef_eff, g.fuse, nch, labels_out, dists_out, stats_out);
  MultiBatch mb;
  bool flagged;
  ANNB_TRY(enqueue_batch(h, 0, true, queries, tables, in_space, B, normalize, k, ef_eff, &g, 1, nullptr, nullptr, filter_labels,
                         filter_space, n_filter, pf ? pf->bits : nullptr, labels_out, dists_out, out_space, stats_out, mb, &flagged));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  return finish_batch(h, mb, flagged, true);
}

extern "C" {

int annb_scan_subset(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k,
                     const uint64_t *subset_labels, int64_t n_subset, uint64_t *labels_out, float *dists_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if (!queries || !labels_out || !dists_out || B < 0 || k <= 0 || n_subset < 0 || (n_subset > 0 && !subset_labels))
    ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  if (B == 0) return ANNB_OK;
  HostGraph &g = h->g;
  const size_t crow = g.code_row_bytes;
  std::vector<uint8_t> codes;
  std::vector<uint64_t> labs;
  codes.reserve((size_t)n_subset * crow);
  labs.reserve((size_t)n_subset);
  for (int64_t i = 0; i < n_subset; i++) {
    auto it = g.label_lookup.find(subset_labels[i]);
    if (it == g.label_lookup.end() || g.deleted(it->second)) continue;
    const uint8_t *c = g.code(it->second);
    codes.insert(codes.end(), c, c + crow);
    labs.push_back(subset_labels[i]);
  }
  const int64_t n = (int64_t)labs.size();
  // the scan works on the handle's flat code matrix: keep the caller's one (annb_set_codes) intact
  uint8_t *saved_codes = h->d_codes;
  const int64_t saved_n = h->n_codes;
  h->d_codes = nullptr;
  h->n_codes = 0;
  int rc = ANNB_OK;
  std::vector<int64_t> ids((size_t)B * k);
  if (n > 0) {
    cudaError_t ce = cudaMalloc(&h->d_codes, (size_t)n * crow + 16);
    if (ce != cudaSuccess) rc = ANNB_ENOMEM;
    if (rc == ANNB_OK && cudaMemcpyAsync(h->d_codes, codes.data(), (size_t)n * crow, cudaMemcpyHostToDevice, h->stream) != cudaSuccess)
      rc = ANNB_ECUDA;
    h->n_codes = n;
    float *t = nullptr, *dd = nullptr;
    int64_t *dids = nullptr;
    const int64_t step = table_chunk_rows(h, B);
    if (rc == ANNB_OK) rc = annb_scratch(h, S_TABLES, (size_t)std::min(step, B) * h->M * h->Ks * sizeof(float), (void **)&t);
    if (rc == ANNB_OK) rc = annb_scratch(h, S_OUT_L, (size_t)B * k * sizeof(int64_t), (void **)&dids);
    if (rc == ANNB_OK) rc = annb_scratch(h, S_OUT_D, (size_t)B * k * sizeof(float), (void **)&dd);
    for (int64_t b0 = 0; b0 < B && rc == ANNB_OK; b0 += step) {
      const int64_t nb = std::min(step, B - b0);
      rc = build_tables(h, queries + (size_t)b0 * h->dim, in_space, nb, normalize, t);
      if (rc == ANNB_OK) rc = launch_scan_topk(h, t, nb, k, dids + b0 * k, dd + b0 * k);
    }
    if (rc == ANNB_OK) {
      cudaMemcpyAsync(ids.data(), dids, (size_t)B * k * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream);
      cudaMemcpyAsync(dists_out, dd, (size_t)B * k * sizeof(float), cudaMemcpyDeviceToHost, h->stream);
      if (cudaStreamSynchronize(h->stream) != cudaSuccess) rc = ANNB_ECUDA;
    }
    if (h->d_codes) cudaFree(h->d_codes);
  }
  h->d_codes = saved_codes;
  h->n_codes = saved_n;
  if (rc == ANNB_ECUDA) annb_set_error("CUDA error in annb_scan_subset: %s", cudaGetErrorString(cudaGetLastError()));
  if (rc == ANNB_ENOMEM) annb_set_error("cudaMalloc failed in annb_scan_subset");
  if (rc != ANNB_OK) return rc;
  for (int64_t i = 0; i < B * k; i++) {
    if (n > 0 && ids[i] >= 0) {
      labels_out[i] = labs[(size_t)ids[i]];
    } else {
      labels_out[i] = UINT64_MAX;
      dists_out[i] = std::numeric_limits<float>::infinity();
    }
  }
  if (n < k) ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  return ANNB_OK;
}

// ---- streaming submit / wait ---------------------------------------------------------------------
// A filtered / deletion-aware batch whose walk flagged queries (found = -1: N outgrew its capacity) is finished at
// wait time: exactly those queries are re-run on the bitmap walk, on the lane's own stream and scratch.
static int lane_finish(annb_index *h, int lane, bool check) {
  annb_index::AsyncLane &L = h->lanes[lane];
  cudaStream_t saved = h->stream;
  h->stream = lane ? h->stream2 : saved;
  const int rc = finish_batch(h, L.batch, L.flagged, check);
  h->stream = saved;
  return rc;
}

static int lane_wait(annb_index *h, int lane) {
  annb_index::AsyncLane &L = h->lanes[lane];
  if (!L.busy) return ANNB_OK;
  ANNB_CUDA(cudaStreamSynchronize(lane ? h->stream2 : h->stream));
  L.busy = false;
  return lane_finish(h, lane, true);
}

static int multi_plan(annb_index *h, int64_t B, int ef_eff, const int *query_filter, std::vector<uint32_t> &perm,
                      std::vector<const uint32_t *> &qf, MultiGroup grp[3]);

// one batch, enqueued entirely on the next ticket's lane (enqueue_batch) once that lane's previous batch is done.  The
// filter is a label list or a prepared bitmap (pf), as in search_impl, or one prepared filter per query (query_filter),
// as in annb_search_multi.
static int submit_impl(annb_index *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                       const uint64_t *filter_labels, int filter_space, int64_t n_filter, const PreparedFilter *pf,
                       const int *query_filter, uint64_t *labels_out, float *dists_out, int out_space, int *ticket_out) {
  if (pf) n_filter = pf->count;
  if (!queries || !labels_out || !dists_out || !ticket_out || B <= 0 || k <= 0 || ef <= 0) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  if (n_filter < 0 || (n_filter > 0 && !filter_labels && !pf)) ANNB_FAIL(ANNB_EINVAL, "bad filter");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  if (!h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  if (h->opt_force_general == 2) ANNB_FAIL(ANNB_EINVAL, "streamed searches do not run on the bitmap walk: use annb_search");
  if (h->dev_dirty || h->deleted_dirty || h->patch_pending) {  // re-upload of the graph: nothing may be in flight
    ANNB_TRY(lane_wait(h, 0));
    ANNB_TRY(lane_wait(h, 1));
    ANNB_TRY(sync_device_graph(h));
  }
  if (h->gd.n == 0) ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  const int ef_eff = std::max(ef, k);
  if (ef_eff > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "max(ef, k)=%d exceeds ANNB_MAX_EF=%d", ef_eff, ANNB_MAX_EF);
  std::vector<uint32_t> perm;
  std::vector<const uint32_t *> qf;
  MultiGroup grp[3];
  if (query_filter) ANNB_TRY(multi_plan(h, B, ef_eff, query_filter, perm, qf, grp));
  else grp[0] = single_group(h, B, ef_eff, filter_labels || pf, n_filter);
  const int ticket = (int)(h->next_ticket++ & 0x3fffffff);
  const int lane = ticket & 1;
  ANNB_TRY(lane_wait(h, lane));  // a lane holds one batch at a time
  annb_index::AsyncLane &L = h->lanes[lane];
  cudaStream_t saved = h->stream;
  h->stream = lane ? h->stream2 : saved;
  bool flagged = false;
  const int rc = enqueue_batch(h, lane, false, queries, nullptr, in_space, B, normalize, k, ef_eff, grp, query_filter ? 3 : 1,
                               query_filter ? &perm : nullptr, query_filter ? &qf : nullptr, filter_labels, filter_space, n_filter,
                               pf ? pf->bits : nullptr, labels_out, dists_out, out_space, nullptr, L.batch, &flagged);
  h->stream = saved;
  if (rc != ANNB_OK) return rc;
  L.busy = true;
  L.flagged = flagged;
  *ticket_out = ticket;
  return ANNB_OK;
}

int annb_search_submit(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                       uint64_t *labels_out, float *dists_out, int out_space, int *ticket_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  return submit_impl(h, queries, in_space, B, normalize, k, ef, nullptr, ANNB_HOST, 0, nullptr, nullptr, labels_out, dists_out,
                     out_space, ticket_out);
}

int annb_search_submit_filtered(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                                const uint64_t *filter_labels, int filter_space, int64_t n_filter, uint64_t *labels_out,
                                float *dists_out, int out_space, int *ticket_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!filter_labels && n_filter != 0) ANNB_FAIL(ANNB_EINVAL, "bad filter");
  return submit_impl(h, queries, in_space, B, normalize, k, ef, filter_labels, filter_space, n_filter, nullptr, nullptr, labels_out,
                     dists_out, out_space, ticket_out);
}

int annb_search_wait(annb_index_t *h, int ticket) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (ticket < 0) ANNB_FAIL(ANNB_EINVAL, "bad ticket");
  return lane_wait(h, ticket & 1);
}

int annb_merge_topk(annb_index_t *h, const uint64_t *labels_gbk, const float *dists_gbk, int G, int64_t B, int k,
                    uint64_t *labels_out, float *dists_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!labels_gbk || !dists_gbk || !labels_out || !dists_out || G <= 0 || k <= 0 || B < 0) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  return launch_merge_topk(h, labels_gbk, dists_gbk, G, B, k, B * (int64_t)k, B * (int64_t)k, labels_out, dists_out, h->stream);
}

int annb_merge_topk_packed(annb_index_t *h, const void *packed, int G, int64_t B, int k, int64_t rank_stride_bytes,
                           int64_t labels_offset_bytes, uint64_t *labels_out, float *dists_out, int lane) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!packed || !labels_out || !dists_out || G <= 0 || k <= 0 || B < 0 || lane < 0 || lane > 1)
    ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  if ((rank_stride_bytes & 7) || (labels_offset_bytes & 7) || labels_offset_bytes < B * (int64_t)k * 4 ||
      rank_stride_bytes < labels_offset_bytes + B * (int64_t)k * 8 || (reinterpret_cast<uintptr_t>(packed) & 7))
    ANNB_FAIL(ANNB_EINVAL, "packed shard results: offsets must be 8-byte aligned and hold (B,k) fp32 + (B,k) u64");
  const float *d = reinterpret_cast<const float *>(packed);
  const uint64_t *l = reinterpret_cast<const uint64_t *>(reinterpret_cast<const uint8_t *>(packed) + labels_offset_bytes);
  return launch_merge_topk(h, l, d, G, B, k, rank_stride_bytes / 8, rank_stride_bytes / 4, labels_out, dists_out,
                           lane ? h->stream2 : h->stream);
}

int annb_lane_stream(annb_index_t *h, int lane, uint64_t *stream_out) {
  if (!h || !stream_out || lane < 0 || lane > 1) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  *stream_out = (uint64_t)(uintptr_t)(lane ? h->stream2 : h->stream);
  return ANNB_OK;
}

int annb_last_kernel_ms(annb_index_t *h, float *table_ms, float *search_ms, float *scan_ms) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  float v;
  if (table_ms) *table_ms = (cudaEventElapsedTime(&v, h->ev[0], h->ev[1]) == cudaSuccess) ? v : -1.f;
  if (search_ms) *search_ms = (cudaEventElapsedTime(&v, h->ev[2], h->ev[3]) == cudaSuccess) ? v : -1.f;
  if (scan_ms) *scan_ms = (cudaEventElapsedTime(&v, h->ev[4], h->ev[5]) == cudaSuccess) ? v : -1.f;
  cudaGetLastError();
  return ANNB_OK;
}

int annb_launch_count(annb_index_t *h, int64_t *out) {
  if (!h || !out) ANNB_FAIL(ANNB_EINVAL, "null argument");
  *out = h->launches;
  return ANNB_OK;
}

int annb_fallback_count(annb_index_t *h, int64_t *out) {
  if (!h || !out) ANNB_FAIL(ANNB_EINVAL, "null argument");
  *out = h->flagged_fallbacks;
  return ANNB_OK;
}

int annb_sync_counts(annb_index_t *h, int64_t *full_syncs, int64_t *patches) {
  if (!h) ANNB_FAIL(ANNB_EINVAL, "null argument");
  if (full_syncs) *full_syncs = h->full_syncs;
  if (patches) *patches = h->patches;
  return ANNB_OK;
}

int annb_device_graph_layout(annb_index_t *h, int64_t *rec0_bytes, int64_t *code_bytes_per_node, int *wide) {
  if (!h) ANNB_FAIL(ANNB_EINVAL, "null argument");
  const bool w = wide_rows(h);
  if (rec0_bytes) *rec0_bytes = h->gd.rec0_bytes;
  if (code_bytes_per_node) *code_bytes_per_node = w ? wide_code_stride(h) : 0;
  if (wide) *wide = w ? 1 : 0;
  return ANNB_OK;
}

static_assert(ANNB_GRAPH_MAX_LEVELS == ANNB_MAX_LEVELS, "annb_device_graph_export's header holds GraphDev::up_off");
static_assert(sizeof(GraphDev::ep_code) == 128, "annb_device_graph_export's header ends with the 128 bytes of ep_code");

int annb_device_graph_export(annb_index_t *h, int part, void *dst, int64_t cap, int64_t *bytes) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!bytes || cap < 0 || (cap > 0 && !dst)) ANNB_FAIL(ANNB_EINVAL, "null bytes / dst, or cap < 0");
  // whatever is still walking or uploading on either lane finishes first (the copies below are synchronous)
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream2));
  const GraphDev &d = h->gd;
  const int64_t n = d.n;
  const bool wide = wide_rows(h);
  const void *src = nullptr;  // device
  size_t size = 0;
  std::vector<uint8_t> head;  // host
  switch (part) {
    case ANNB_GRAPH_PART_HEADER: {
      const int64_t f[14] = {d.n, d.maxlevel, d.ep_node, d.ep_rec, d.maxM, d.maxM0, d.code_row, d.rec0_bytes, d.code_off0,
                             d.recu_bytes, d.code_offu, d.tail_offu, (int64_t)h->max_label, h->labels_identity ? 1 : 0};
      head.resize(ANNB_GRAPH_HEADER_BYTES);
      memcpy(head.data(), f, sizeof(f));
      for (int l = 0; l < ANNB_MAX_LEVELS; l++) {
        const int64_t o = (int64_t)d.up_off[l];
        memcpy(head.data() + sizeof(f) + 8 * l, &o, 8);
      }
      memcpy(head.data() + sizeof(f) + 8 * ANNB_MAX_LEVELS, d.ep_code, sizeof(d.ep_code));
      size = head.size();
      break;
    }
    case ANNB_GRAPH_PART_REC0: src = d.rec0; size = d.rec0 ? (size_t)n * d.rec0_bytes : 0; break;
    case ANNB_GRAPH_PART_UPPER: src = d.up; size = d.up ? h->up_bytes : 0; break;
    case ANNB_GRAPH_PART_LABELS: src = d.labels; size = d.labels ? (size_t)n * 8 : 0; break;
    case ANNB_GRAPH_PART_DELETED: src = d.deleted; size = d.deleted ? ((size_t)(n + 31) / 32 + 1) * 4 : 0; break;
    case ANNB_GRAPH_PART_WIDE_CODES:
      src = h->d_wide_codes;
      size = wide && h->d_wide_codes ? (size_t)n * wide_code_stride(h) : 0;
      break;
    case ANNB_GRAPH_PART_OWN_CODES:
      src = h->d_own_codes;
      size = h->d_own_codes && h->own_codes_gen == h->state_gen ? (size_t)h->g.count.load() * h->g.code_row_bytes : 0;
      break;
    default: ANNB_FAIL(ANNB_EINVAL, "unknown device graph part %d", part);
  }
  *bytes = (int64_t)size;
  const size_t c = std::min(size, (size_t)cap);
  if (c == 0) return ANNB_OK;
  if (!head.empty()) memcpy(dst, head.data(), c);
  else ANNB_CUDA(cudaMemcpy(dst, src, c, cudaMemcpyDeviceToHost));
  return ANNB_OK;
}

int annb_fallback_queries(annb_index_t *h, int64_t *out) {
  if (!h || !out) ANNB_FAIL(ANNB_EINVAL, "null argument");
  *out = h->flagged_fallback_queries;
  return ANNB_OK;
}

int annb_set_option(annb_index_t *h, const char *name, int64_t value) {
  ANNB_ENTER(h);
  if (!name) ANNB_FAIL(ANNB_EINVAL, "null option name");
  if (!strcmp(name, "warps_per_cta")) h->opt_warps_per_cta = value;
  else if (!strcmp(name, "ctas_per_sm")) h->opt_ctas_per_sm = value;
  else if (!strcmp(name, "force_general")) h->opt_force_general = value;
  else if (!strcmp(name, "timing")) h->opt_timing = value;
  else if (!strcmp(name, "ip_raw")) h->opt_ip_raw = value;
  else if (!strcmp(name, "chunks")) h->opt_chunks = value;
  else if (!strcmp(name, "flagged_epl")) h->opt_flagged_epl = value;
  else if (!strcmp(name, "flagged_kernel")) h->opt_flagged_kernel = value;
  else if (!strcmp(name, "flagged_en")) h->opt_flagged_en = value;
  else if (!strcmp(name, "scan_kernel")) h->opt_scan_kernel = value;
  else if (!strcmp(name, "subset_chunk_rows")) h->opt_subset_chunk_rows = value;
  else if (!strcmp(name, "walk_kernel")) h->opt_walk_kernel = value;
  else if (!strcmp(name, "dump_tables")) h->opt_dump_tables = value;
  else if (!strcmp(name, "gpu_build")) h->opt_gpu_build = value;
  else if (!strcmp(name, "gpu_build_frac")) h->opt_gpu_build_frac = value;
  else if (!strcmp(name, "reset_counters")) h->flagged_fallbacks = h->flagged_fallback_queries = 0;
  else ANNB_FAIL(ANNB_EINVAL, "unknown option %s", name);
  return ANNB_OK;
}

}  // extern "C"

// ---- attribute columns and prepared filters ----------------------------------------------------------
static int drain_lanes(annb_index *h) {  // streamed searches in flight finish before anything they read changes
  if (h->device < 0) return ANNB_OK;
  ANNB_TRY(settle_flagged_lanes(h));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream2));
  return ANNB_OK;
}

static int attr_width(int type) { return type == ANNB_ATTR_TEXT ? 4 : 8; }

// structural checks of a filter program; nothing runs before it passes
static int validate_program(const annb_index *h, const annb_filter_op_t *prog, int n_ops, const void *consts,
                            int64_t n_const_bytes) {
  if (n_ops <= 0 || !prog) ANNB_FAIL(ANNB_EINVAL, "filter program is empty");
  if (n_ops > ANNB_FILTER_MAX_OPS) ANNB_FAIL(ANNB_ELIMIT, "filter program has %d ops (limit %d)", n_ops, ANNB_FILTER_MAX_OPS);
  if (n_const_bytes < 0 || (n_const_bytes > 0 && !consts) || n_const_bytes % 8)
    ANNB_FAIL(ANNB_EINVAL, "filter constants: size must be a multiple of 8 bytes");
  if (n_const_bytes > ANNB_FILTER_MAX_CONST_BYTES)
    ANNB_FAIL(ANNB_ELIMIT, "filter constants take %lld bytes (limit %d)", (long long)n_const_bytes, ANNB_FILTER_MAX_CONST_BYTES);
  int depth = 0;
  for (int i = 0; i < n_ops; i++) {
    const annb_filter_op_t &o = prog[i];
    if (o.op < ANNB_FOP_FALSE || o.op > ANNB_FOP_OR) ANNB_FAIL(ANNB_EINVAL, "filter op %d: unknown op code %d", i, o.op);
    if (o.op == ANNB_FOP_AND || o.op == ANNB_FOP_OR) {
      if (depth < 2) ANNB_FAIL(ANNB_EINVAL, "filter op %d: AND / OR needs two operands", i);
      depth--;
      continue;
    }
    if (++depth > ANNB_FILTER_MAX_DEPTH) ANNB_FAIL(ANNB_ELIMIT, "filter program nests deeper than %d", ANNB_FILTER_MAX_DEPTH);
    if (o.op == ANNB_FOP_FALSE || o.op == ANNB_FOP_TRUE) continue;
    if (o.col < 0 || o.col >= (int)h->attrs.size() || h->attrs[o.col].type < 0)
      ANNB_FAIL(ANNB_EINVAL, "filter op %d: no attribute column %d", i, o.col);
    const int type = h->attrs[o.col].type;
    int want = -1;
    int64_t need = 0, align = 8;
    switch (o.op) {
      case ANNB_FOP_NOTNULL: want = type; break;
      case ANNB_FOP_INT_RANGE: want = ANNB_ATTR_INTEGER; need = 16; break;
      case ANNB_FOP_INT_NE: want = ANNB_ATTR_INTEGER; need = 8; break;
      case ANNB_FOP_INT_IN: case ANNB_FOP_INT_NIN: want = ANNB_ATTR_INTEGER; need = 8 * (int64_t)o.b; break;
      case ANNB_FOP_FLT_RANGE: want = ANNB_ATTR_FLOAT; need = 16; break;
      case ANNB_FOP_FLT_NE: want = ANNB_ATTR_FLOAT; need = 8; break;
      case ANNB_FOP_FLT_IN: case ANNB_FOP_FLT_NIN: want = ANNB_ATTR_FLOAT; need = 8 * (int64_t)o.b; break;
      case ANNB_FOP_CODE_IN: want = ANNB_ATTR_TEXT; need = 4 * (((int64_t)o.b + 31) / 32); align = 4; break;
    }
    if (type != want) ANNB_FAIL(ANNB_EINVAL, "filter op %d: op %d does not apply to column %d of type %d", i, o.op, o.col, type);
    if (o.b < 0) ANNB_FAIL(ANNB_EINVAL, "filter op %d: negative count", i);
    if (o.op != ANNB_FOP_NOTNULL && (o.a < 0 || o.a % align || (int64_t)o.a + need > n_const_bytes))
      ANNB_FAIL(ANNB_EINVAL, "filter op %d: constants [%d, %lld) outside the pool of %lld bytes or misaligned", i, o.a,
                (long long)o.a + need, (long long)n_const_bytes);
    // the evaluator's membership test is a binary search: a list must be non-decreasing, and a FLOAT one free of NaN
    const bool int_list = o.op == ANNB_FOP_INT_IN || o.op == ANNB_FOP_INT_NIN;
    if (int_list || o.op == ANNB_FOP_FLT_IN || o.op == ANNB_FOP_FLT_NIN) {
      const uint8_t *k = (const uint8_t *)consts + o.a;
      for (int j = 0; j < o.b; j++) {
        int64_t iv, ip = 0;
        double dv, dp = 0.0;
        memcpy(&iv, k + 8 * j, 8);
        memcpy(&dv, k + 8 * j, 8);
        if (j) {
          memcpy(&ip, k + 8 * (j - 1), 8);
          memcpy(&dp, k + 8 * (j - 1), 8);
        }
        if (!int_list && std::isnan(dv)) ANNB_FAIL(ANNB_EINVAL, "filter op %d (op code %d): list entry %d is NaN", i, o.op, j);
        if (j && (int_list ? iv < ip : dv < dp))
          ANNB_FAIL(ANNB_EINVAL, "filter op %d (op code %d): list is not sorted ascending at entry %d", i, o.op, j);
      }
    }
  }
  if (depth != 1) ANNB_FAIL(ANNB_EINVAL, "filter program leaves %d values on the stack (must be 1)", depth);
  return ANNB_OK;
}

// bring the device copy of a column up to date for rows [0, n): the dirty range, new rows, or all of it after a
// reallocation
static int attr_sync_dev(annb_index *h, AttrColumn &c, int64_t n) {
  const size_t words = (size_t)(n + 31) / 32 + 1;
  const size_t vbytes = (size_t)std::max<int64_t>(n, 1) * c.width;
  int64_t lo = std::min(c.dirty_lo, c.dev_rows), hi = std::max(c.dirty_hi, n);
  if (c.cap_vals < vbytes || c.cap_valid < words * 4 || !c.d_vals || !c.d_valid) {
    ANNB_TRY(ensure_dev((void **)&c.d_vals, &c.cap_vals, vbytes));
    ANNB_TRY(ensure_dev((void **)&c.d_valid, &c.cap_valid, words * 4));
    lo = 0;
  }
  hi = std::min(hi, n);
  if (hi > lo) {
    ANNB_CUDA(cudaMemcpyAsync(c.d_vals + (size_t)lo * c.width, c.vals.data() + (size_t)lo * c.width, (size_t)(hi - lo) * c.width,
                              cudaMemcpyHostToDevice, h->stream));
  }
  const size_t w0 = (size_t)std::max<int64_t>(lo, 0) / 32, w1 = words;  // validity: from the first dirty word to the end
  if (w1 > w0)
    ANNB_CUDA(cudaMemcpyAsync(c.d_valid + w0, c.valid.data() + w0, (w1 - w0) * 4, cudaMemcpyHostToDevice, h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));  // the host vectors may be written again as soon as this returns
  c.dev_rows = n;
  c.dirty_lo = std::numeric_limits<int64_t>::max();
  c.dirty_hi = 0;
  return ANNB_OK;
}

static int find_filter(annb_index *h, int filter_id, PreparedFilter **out) {
  auto it = h->filters.find(filter_id);
  if (it == h->filters.end()) ANNB_FAIL(ANNB_EINVAL, "no prepared filter %d", filter_id);
  if (it->second.gen != h->state_gen)
    ANNB_FAIL(ANNB_ESTATE, "prepared filter %d is stale: the graph, the deletions or the attributes changed since it was prepared",
              filter_id);
  *out = &it->second;
  return ANNB_OK;
}

// F programs given back to back -> F prepared filters.  Everything is validated first; the referenced columns are
// synced once; the programs are packed into as few evaluator launches as the LAUNCH limits allow (a launch of one
// program takes filter_eval_kernel<false>, the single-filter kernel), all uploaded in one copy; one synchronisation.
// The F bitmaps share one allocation.
static int prepare_many_impl(annb_index *h, int F, const annb_filter_op_t *programs, const int *n_ops, const void *consts,
                             const int64_t *n_const_bytes, int *filter_ids, int64_t *counts) {
  std::vector<int64_t> op0((size_t)F + 1, 0), c0((size_t)F + 1, 0);
  for (int f = 0; f < F; f++) {
    if (n_ops[f] < 0 || n_const_bytes[f] < 0) ANNB_FAIL(ANNB_EINVAL, "filter %d: negative size", f);
    op0[f + 1] = op0[f] + n_ops[f];
    c0[f + 1] = c0[f] + n_const_bytes[f];
  }
  const uint8_t *cbase = (const uint8_t *)consts;
  for (int f = 0; f < F; f++) {
    if (n_const_bytes[f] > 0 && !consts) ANNB_FAIL(ANNB_EINVAL, "filter %d: null constants", f);
    const int rc = validate_program(h, programs + op0[f], n_ops[f], n_const_bytes[f] ? cbase + c0[f] : nullptr, n_const_bytes[f]);
    if (rc != ANNB_OK) {
      if (F > 1) {
        const std::string msg = annb_last_error();
        annb_set_error("filter %d: %s", f, msg.c_str());
      }
      return rc;
    }
  }
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  ANNB_TRY(drain_lanes(h));
  ANNB_TRY(sync_device_graph(h));
  attr_fit(h);
  const int64_t n = h->gd.n;
  std::vector<AttrColDev> cols(h->attrs.size());
  std::vector<char> used(h->attrs.size(), 0);
  for (int64_t i = 0; i < op0[F]; i++)
    if (programs[i].op != ANNB_FOP_AND && programs[i].op != ANNB_FOP_OR && programs[i].op > ANNB_FOP_TRUE) used[programs[i].col] = 1;
  for (size_t c = 0; c < h->attrs.size(); c++) {
    if (!used[c]) continue;
    ANNB_TRY(attr_sync_dev(h, h->attrs[c], n));
    cols[c] = AttrColDev{h->attrs[c].d_vals, h->attrs[c].d_valid, h->attrs[c].type};
  }
  // launches: consecutive programs while their ops and constants fit one launch's shared memory (a single program
  // always fits: ANNB_FILTER_MAX_OPS / _CONST_BYTES are below the LAUNCH limits)
  struct Launch {
    int f0, f1;
    size_t prog, offs, consts;  // byte offsets in the upload
    int ops, cbytes;
  };
  auto up16 = [](size_t x) { return (x + 15) / 16 * 16; };
  std::vector<Launch> launches;
  for (int f = 0; f < F;) {
    Launch l{f, f, 0, 0, 0, 0, 0};
    while (l.f1 < F && (l.f1 == l.f0 || (l.ops + n_ops[l.f1] <= ANNB_FILTER_LAUNCH_MAX_OPS &&
                                          l.cbytes + n_const_bytes[l.f1] <= ANNB_FILTER_LAUNCH_MAX_CONST_BYTES))) {
      l.ops += n_ops[l.f1];
      l.cbytes += (int)n_const_bytes[l.f1];
      l.f1++;
    }
    launches.push_back(l);
    f = l.f1;
  }
  size_t total = 0;
  for (Launch &l : launches) {
    l.prog = total;
    total = up16(total + (size_t)l.ops * sizeof(annb_filter_op_t));
    l.consts = total;
    total = up16(total + (size_t)l.cbytes);
    l.offs = total;
    total = up16(total + (size_t)(l.f1 - l.f0 + 1) * 4);
  }
  const size_t counts_at = total;
  total += (size_t)F * 8;
  std::vector<uint8_t> up(total, 0);
  for (const Launch &l : launches) {
    annb_filter_op_t *dst = reinterpret_cast<annb_filter_op_t *>(up.data() + l.prog);
    int *offs = reinterpret_cast<int *>(up.data() + l.offs);
    int at = 0, cat = 0;
    for (int f = l.f0; f < l.f1; f++) {
      offs[f - l.f0] = at;
      for (int i = 0; i < n_ops[f]; i++) {
        annb_filter_op_t o = programs[op0[f] + i];
        if (o.op >= ANNB_FOP_INT_RANGE && o.op <= ANNB_FOP_CODE_IN) o.a += cat;  // into the launch's one pool
        dst[at++] = o;
      }
      if (n_const_bytes[f]) memcpy(up.data() + l.consts + cat, cbase + c0[f], (size_t)n_const_bytes[f]);
      cat += (int)n_const_bytes[f];
    }
    offs[l.f1 - l.f0] = at;
  }
  uint8_t *dbuf;
  ANNB_TRY(annb_scratch(h, S_FILTER_PROG, total, (void **)&dbuf));
  unsigned long long *dcounts = (unsigned long long *)(dbuf + counts_at);
  const int64_t words = (n + 31) / 32 + 1, stride = (words + 3) / 4 * 4;  // bitmaps 16-byte aligned
  void *block = nullptr;
  ANNB_CUDA(cudaMalloc(&block, (size_t)stride * 4 * F));
  std::shared_ptr<void> owner(block, [](void *p) { cudaFree(p); });
  uint32_t *bits = (uint32_t *)block;
  int rc = ANNB_OK;
  std::vector<unsigned long long> hcounts((size_t)F, 0);
  if (cudaMemcpyAsync(dbuf, up.data(), counts_at, cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
      cudaMemsetAsync(dcounts, 0, (size_t)F * 8, h->stream) != cudaSuccess)
    rc = ANNB_ECUDA;
  for (size_t i = 0; i < launches.size() && rc == ANNB_OK; i++) {
    const Launch &l = launches[i];
    const annb_filter_op_t *dprog = (const annb_filter_op_t *)(dbuf + l.prog);
    if (l.f1 - l.f0 == 1)
      rc = launch_filter_eval(h, dprog, l.ops, dbuf + l.consts, l.cbytes, cols.data(), (int)cols.size(), n, h->gd.deleted,
                              bits + (size_t)l.f0 * stride, dcounts + l.f0);
    else
      rc = launch_filter_eval_many(h, l.f1 - l.f0, dprog, (const int *)(dbuf + l.offs), l.ops, dbuf + l.consts, l.cbytes, cols.data(),
                                   (int)cols.size(), n, h->gd.deleted, bits + (size_t)l.f0 * stride, stride, dcounts + l.f0);
  }
  if (rc == ANNB_OK && (cudaMemcpyAsync(hcounts.data(), dcounts, (size_t)F * 8, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
                        cudaStreamSynchronize(h->stream) != cudaSuccess))
    rc = ANNB_ECUDA;
  if (rc != ANNB_OK) {
    if (rc == ANNB_ECUDA) annb_set_error("CUDA error while evaluating a filter: %s", cudaGetErrorString(cudaGetLastError()));
    return rc;
  }
  for (int f = 0; f < F; f++) {
    PreparedFilter pf;
    pf.bits = bits + (size_t)f * stride;
    pf.block = owner;
    pf.n = n;
    pf.count = (int64_t)hcounts[f];
    pf.gen = h->state_gen;
    const int id = h->next_filter_id++;
    h->filters[id] = pf;
    filter_ids[f] = id;
    counts[f] = pf.count;
  }
  return ANNB_OK;
}

// the cell sets (cells.cu) use a cell's prepared filters under that cell's lock
int find_prepared_filter(annb_index *h, int filter_id, PreparedFilter **out) { return find_filter(h, filter_id, out); }

// The walk layout keeps a node's code only in its neighbours' records; the exact subset scan reads each node's own code
// from this copy of the host graph's, re-made after any change (state_gen) on the first scan that needs it.
int sync_own_codes(annb_index *h, const uint8_t **out) {
  HostGraph &g = h->g;
  const int64_t n = g.count.load();
  const size_t crow = g.code_row_bytes;
  if (!h->d_own_codes || h->own_codes_gen != h->state_gen) {
    std::vector<uint8_t> hc((size_t)n * crow);
    for (int64_t i = 0; i < n; i++) memcpy(hc.data() + (size_t)i * crow, g.code((uint32_t)i), crow);
    ANNB_TRY(ensure_dev((void **)&h->d_own_codes, &h->cap_own_codes, std::max<size_t>(hc.size(), 16)));
    if (n) ANNB_CUDA(cudaMemcpy(h->d_own_codes, hc.data(), hc.size(), cudaMemcpyHostToDevice));
    h->own_codes_gen = h->state_gen;
  }
  *out = h->d_own_codes;
  return ANNB_OK;
}

// annb_search_prepared with the (B, 3) counters of annb_search; takes the handle's lock
int search_prepared_stats(annb_index *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef, int filter_id,
                          uint64_t *labels_out, float *dists_out, int out_space, int64_t *stats_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  PreparedFilter *f;
  ANNB_TRY(find_filter(h, filter_id, &f));
  return search_impl(h, queries, nullptr, in_space, B, normalize, k, ef, nullptr, ANNB_HOST, 0, f, labels_out, dists_out, out_space,
                     stats_out);
}

extern "C" {

int annb_attr_define(annb_index_t *h, int col, int type) {
  ANNB_ENTER(h);
  if (type < ANNB_ATTR_INTEGER || type > ANNB_ATTR_TEXT) ANNB_FAIL(ANNB_EINVAL, "unknown attribute type %d", type);
  if (col < 0 || col >= ANNB_MAX_ATTR_COLUMNS) ANNB_FAIL(ANNB_ELIMIT, "attribute column %d (limit %d columns)", col, ANNB_MAX_ATTR_COLUMNS);
  if (col < (int)h->attrs.size()) {
    if (h->attrs[col].type != type) ANNB_FAIL(ANNB_EINVAL, "attribute column %d is already declared with type %d", col, h->attrs[col].type);
    return ANNB_OK;
  }
  if (col != (int)h->attrs.size()) ANNB_FAIL(ANNB_EINVAL, "attribute columns are declared in order: next is %d", (int)h->attrs.size());
  h->attrs.emplace_back();
  h->attrs.back().type = type;
  h->attrs.back().width = attr_width(type);
  h->attrs.back().dirty_lo = 0;
  h->attrs.back().dirty_hi = std::numeric_limits<int64_t>::max();
  attr_fit(h);
  h->state_gen++;
  return ANNB_OK;
}

int annb_attr_set(annb_index_t *h, int col, const uint64_t *labels, int64_t n, const void *values, const uint8_t *valid, int space) {
  ANNB_ENTER(h);
  if (col < 0 || col >= (int)h->attrs.size()) ANNB_FAIL(ANNB_EINVAL, "no attribute column %d", col);
  if (n < 0 || (n > 0 && (!labels || !values))) ANNB_FAIL(ANNB_EINVAL, "null labels / values");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  if (n == 0) return ANNB_OK;
  AttrColumn &c = h->attrs[col];
  std::vector<uint64_t> hl;
  std::vector<uint8_t> hv, hvalid;
  if (space == ANNB_DEVICE) {
    ANNB_NEED_GPU(h);
    hl.resize((size_t)n);
    hv.resize((size_t)n * c.width);
    ANNB_CUDA(cudaMemcpy(hl.data(), labels, (size_t)n * 8, cudaMemcpyDeviceToHost));
    ANNB_CUDA(cudaMemcpy(hv.data(), values, (size_t)n * c.width, cudaMemcpyDeviceToHost));
    labels = hl.data();
    values = hv.data();
    if (valid) {
      hvalid.resize((size_t)n);
      ANNB_CUDA(cudaMemcpy(hvalid.data(), valid, (size_t)n, cudaMemcpyDeviceToHost));
      valid = hvalid.data();
    }
  }
  std::vector<uint32_t> ids((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    auto it = h->g.label_lookup.find(labels[i]);
    if (it == h->g.label_lookup.end()) ANNB_FAIL(ANNB_ENOTFOUND, "Label not found");
    ids[i] = it->second;
    if (c.type == ANNB_ATTR_TEXT && (!valid || valid[i])) {
      int32_t code;
      memcpy(&code, (const uint8_t *)values + (size_t)i * 4, 4);
      if (code < 0) ANNB_FAIL(ANNB_EINVAL, "TEXT codes must be >= 0 (row %lld has %d)", (long long)i, code);
    }
  }
  ANNB_TRY(drain_lanes(h));
  attr_fit(h);
  for (int64_t i = 0; i < n; i++) {
    const uint32_t id = ids[i];
    const bool ok = !valid || valid[i];
    if (ok) memcpy(c.vals.data() + (size_t)id * c.width, (const uint8_t *)values + (size_t)i * c.width, (size_t)c.width);
    else memset(c.vals.data() + (size_t)id * c.width, 0, (size_t)c.width);
    if (ok) c.valid[id >> 5] |= 1u << (id & 31);
    else c.valid[id >> 5] &= ~(1u << (id & 31));
    c.dirty_lo = std::min<int64_t>(c.dirty_lo, id);
    c.dirty_hi = std::max<int64_t>(c.dirty_hi, (int64_t)id + 1);
  }
  h->state_gen++;
  return ANNB_OK;
}

int annb_attr_export(annb_index_t *h, int col, void *values, uint8_t *valid, int64_t cap, int64_t *n_out) {
  ANNB_ENTER(h);
  if (col < 0 || col >= (int)h->attrs.size()) ANNB_FAIL(ANNB_EINVAL, "no attribute column %d", col);
  if (cap < 0) ANNB_FAIL(ANNB_EINVAL, "negative capacity");
  attr_fit(h);
  const AttrColumn &c = h->attrs[col];
  const int64_t rows = h->g.inited ? h->g.count.load() : 0;
  const int64_t m = std::min(cap, rows);
  if (values && m) memcpy(values, c.vals.data(), (size_t)m * c.width);
  if (valid)
    for (int64_t i = 0; i < m; i++) valid[i] = (uint8_t)((c.valid[i >> 5] >> (i & 31)) & 1u);
  if (n_out) *n_out = rows;
  return ANNB_OK;
}

int annb_attr_clear(annb_index_t *h) {
  ANNB_ENTER(h);
  ANNB_TRY(drain_lanes(h));
  for (AttrColumn &c : h->attrs) {
    if (c.d_vals) cudaFree(c.d_vals);
    if (c.d_valid) cudaFree(c.d_valid);
  }
  h->attrs.clear();
  h->state_gen++;
  return ANNB_OK;
}

int annb_filter_prepare(annb_index_t *h, const annb_filter_op_t *program, int n_ops, const void *consts, int64_t n_const_bytes,
                        int *filter_id, int64_t *count) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!filter_id || !count) ANNB_FAIL(ANNB_EINVAL, "null outputs");
  *filter_id = 0;
  *count = 0;
  return prepare_many_impl(h, 1, program, &n_ops, consts, &n_const_bytes, filter_id, count);
}

int annb_filter_prepare_many(annb_index_t *h, int F, const annb_filter_op_t *programs, const int *n_ops, const void *consts,
                             const int64_t *n_const_bytes, int *filter_ids_out, int64_t *counts_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (F <= 0 || !programs || !n_ops || !n_const_bytes || !filter_ids_out || !counts_out) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  if (F > ANNB_FILTER_MAX_PER_CALL) ANNB_FAIL(ANNB_ELIMIT, "%d filters in one call (limit %d)", F, ANNB_FILTER_MAX_PER_CALL);
  for (int f = 0; f < F; f++) {
    filter_ids_out[f] = 0;
    counts_out[f] = 0;
  }
  return prepare_many_impl(h, F, programs, n_ops, consts, n_const_bytes, filter_ids_out, counts_out);
}

int annb_filter_prepare_labels(annb_index_t *h, const uint64_t *labels, int64_t n, int space, int *filter_id, int64_t *count) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!filter_id || !count || n < 0 || (n > 0 && !labels)) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  *filter_id = 0;
  *count = 0;
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  ANNB_TRY(drain_lanes(h));  // the label staging buffers are lane 0's
  ANNB_TRY(sync_device_graph(h));
  const int64_t rows = h->gd.n;
  const size_t words = (size_t)(rows + 31) / 32 + 1;
  // the entries that name live rows, in order, repeats kept: the subset an exact scan of this list covers
  std::vector<uint64_t> hl;
  const uint64_t *lab = labels;
  if (space == ANNB_DEVICE && n > 0) {
    hl.resize((size_t)n);
    ANNB_CUDA(cudaMemcpy(hl.data(), labels, (size_t)n * 8, cudaMemcpyDeviceToHost));
    lab = hl.data();
  }
  std::vector<uint32_t> ids;
  for (int64_t i = 0; i < n; i++) {
    auto it = h->g.label_lookup.find(lab[i]);
    if (it != h->g.label_lookup.end() && !h->g.deleted(it->second)) ids.push_back(it->second);
  }
  uint64_t *staged;
  uint32_t *by_label;
  ANNB_TRY(label_staging(h, 0, space, n, &staged, &by_label));
  void *block = nullptr;
  ANNB_CUDA(cudaMalloc(&block, (words + ids.size()) * 4));
  std::shared_ptr<void> owner(block, [](void *p) { cudaFree(p); });
  uint32_t *bits = (uint32_t *)block;
  ANNB_CUDA(cudaMemsetAsync(bits, 0, words * 4, h->stream));
  if (!ids.empty()) ANNB_CUDA(cudaMemcpyAsync(bits + words, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, h->stream));
  ANNB_TRY(labels_to_bitmap(h, labels, space, n, staged, by_label, bits));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  PreparedFilter pf;
  pf.bits = bits;
  pf.block = owner;
  pf.n = rows;
  pf.count = n;  // as a label list counts: every entry, repeats and labels not in the graph included
  pf.gen = h->state_gen;
  pf.ids = bits + words;
  pf.n_ids = (int64_t)ids.size();
  const int id = h->next_filter_id++;
  h->filters[id] = pf;
  *filter_id = id;
  *count = n;
  return ANNB_OK;
}

// The rows listed are the bitmap's.  A program's bitmap already excludes deleted rows; a label list's bitmap holds
// every row the list names (the walks test deletions separately), so its deleted rows are masked out here.  Only
// the entries the compaction wrote are copied: their number comes back from the device before anything is copied.
int annb_filter_labels(annb_index_t *h, int filter_id, uint64_t *labels_out, int64_t cap, int64_t *n_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (cap < 0 || (cap > 0 && !labels_out)) ANNB_FAIL(ANNB_EINVAL, "bad output buffer");
  PreparedFilter *f;
  ANNB_TRY(find_filter(h, filter_id, &f));
  if (n_out) *n_out = 0;
  // at most this many rows are listed: a program's count, or a label list's entries that name live rows
  const int64_t bound = std::min(f->n, f->ids ? f->n_ids : f->count);
  if (bound == 0) return ANNB_OK;
  const uint32_t *drop = f->ids ? h->gd.deleted : nullptr;
  const int64_t nb = filter_compact_blocks(f->n);
  unsigned int *dscan, total = 0;
  uint64_t *dout;
  ANNB_TRY(annb_scratch(h, S_FILTER_SCAN, (size_t)(nb + 1) * 4, (void **)&dscan));
  ANNB_TRY(launch_filter_count(h, f->bits, drop, f->n, dscan));
  ANNB_CUDA(cudaMemcpyAsync(&total, dscan + nb, 4, cudaMemcpyDeviceToHost, h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  if (n_out) *n_out = total;
  const int64_t m = std::min<int64_t>(cap, total);
  if (m == 0) return ANNB_OK;
  ANNB_TRY(annb_scratch(h, S_FILTER_OUT, (size_t)total * 8, (void **)&dout));
  ANNB_TRY(launch_filter_compact(h, f->bits, drop, f->n, h->d_labels, dout, dscan));
  ANNB_CUDA(cudaMemcpyAsync(labels_out, dout, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  return ANNB_OK;
}

int annb_filter_release(annb_index_t *h, int filter_id) {
  ANNB_ENTER(h);
  auto it = h->filters.find(filter_id);
  if (it == h->filters.end()) ANNB_FAIL(ANNB_EINVAL, "no prepared filter %d", filter_id);
  ANNB_TRY(drain_lanes(h));  // a streamed batch may still walk (or re-run on) this bitmap
  h->filters.erase(it);      // frees the block once no filter of its prepare call is left
  return ANNB_OK;
}

int annb_search_prepared(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef, int filter_id,
                         uint64_t *labels_out, float *dists_out, int out_space) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  PreparedFilter *f;
  ANNB_TRY(find_filter(h, filter_id, &f));
  return search_impl(h, queries, nullptr, in_space, B, normalize, k, ef, nullptr, ANNB_HOST, 0, f, labels_out, dists_out, out_space,
                     nullptr);
}

int annb_search_submit_prepared(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                                int filter_id, uint64_t *labels_out, float *dists_out, int out_space, int *ticket_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  PreparedFilter *f;
  ANNB_TRY(find_filter(h, filter_id, &f));
  return submit_impl(h, queries, in_space, B, normalize, k, ef, nullptr, ANNB_HOST, 0, f, nullptr, labels_out, dists_out, out_space,
                     ticket_out);
}

// ---- per-query filters ----------------------------------------------------------------------------------
// A batch with one filter per query is split into three routing groups (MultiGroup), gathered into contiguous blocks,
// each on the route annb_search_prepared / annb_search take for the same rows.  Each walk reads query q's bitmap from
// the per-query table; queries any walk flagged are re-run on the bitmap walk with their own bitmap.
static int multi_plan(annb_index *h, int64_t B, int ef_eff, const int *query_filter, std::vector<uint32_t> &perm,
                      std::vector<const uint32_t *> &qf, MultiGroup grp[3]) {
  std::unordered_map<int, std::pair<const PreparedFilter *, int>> seen;  // id -> (filter, group)
  std::vector<int8_t> which((size_t)B);
  std::vector<const uint32_t *> bits((size_t)B, nullptr);
  double smin[3] = {search_selectivity(h, false, 0), 1.0, 1.0};
  int64_t cnt[3] = {0, 0, 0};
  for (int64_t b = 0; b < B; b++) {
    const int id = query_filter[b];
    int g = 0;
    if (id != 0) {
      auto it = seen.find(id);
      if (it == seen.end()) {
        PreparedFilter *pf;
        ANNB_TRY(find_filter(h, id, &pf));
        const double s = search_selectivity(h, true, pf->count);
        bool walk4f;
        search_route(h, ef_eff, true, s, nullptr, &walk4f);
        g = walk4f ? 1 : 2;
        smin[g] = std::min(smin[g], s);
        it = seen.emplace(id, std::make_pair((const PreparedFilter *)pf, g)).first;
      }
      g = it->second.second;
      bits[(size_t)b] = it->second.first->bits;
    }
    which[(size_t)b] = (int8_t)g;
    cnt[g]++;
  }
  int64_t at[3] = {0, cnt[0], cnt[0] + cnt[1]};
  perm.resize((size_t)B);
  qf.resize((size_t)B);
  for (int g = 0; g < 3; g++) {
    grp[g].o = at[g];
    grp[g].n = cnt[g];
    grp[g].filtered = g > 0;
    grp[g].s = smin[g];
    grp[g].mode = search_route(h, ef_eff, g > 0, smin[g], &grp[g].fuse, nullptr);
  }
  for (int64_t b = 0; b < B; b++) {
    const int64_t pos = at[which[(size_t)b]]++;
    perm[(size_t)pos] = (uint32_t)b;
    qf[(size_t)pos] = bits[(size_t)b];
  }
  return ANNB_OK;
}

int annb_search_multi(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                      const int *query_filter, uint64_t *labels_out, float *dists_out, int out_space) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  ANNB_TRY(settle_flagged_lanes(h));
  if (B < 0 || k <= 0 || ef <= 0 || (B > 0 && (!queries || !query_filter || !labels_out || !dists_out)))
    ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  if (!h->d_codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  ANNB_TRY(sync_device_graph(h));
  if (B == 0) return ANNB_OK;
  const int ef_eff = std::max(ef, k);  // hnswalg.h:1279
  if (ef_eff > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "max(ef, k)=%d exceeds ANNB_MAX_EF=%d", ef_eff, ANNB_MAX_EF);
  std::vector<uint32_t> perm;
  std::vector<const uint32_t *> qf;
  MultiGroup grp[3];
  ANNB_TRY(multi_plan(h, B, ef_eff, query_filter, perm, qf, grp));
  if (h->gd.n == 0) ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  MultiBatch mb;
  bool flagged;
  ANNB_TRY(enqueue_batch(h, 0, true, queries, nullptr, in_space, B, normalize, k, ef_eff, grp, 3, &perm, &qf, nullptr, ANNB_HOST, 0,
                         nullptr, labels_out, dists_out, out_space, nullptr, mb, &flagged));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  return finish_batch(h, mb, flagged, true);
}

int annb_search_submit_multi(annb_index_t *h, const float *queries, int in_space, int64_t B, int normalize, int k, int ef,
                             const int *query_filter, uint64_t *labels_out, float *dists_out, int out_space, int *ticket_out) {
  ANNB_ENTER(h);
  ANNB_NEED_GPU(h);
  if (!query_filter) ANNB_FAIL(ANNB_EINVAL, "bad arguments");
  return submit_impl(h, queries, in_space, B, normalize, k, ef, nullptr, ANNB_HOST, 0, nullptr, query_filter, labels_out, dists_out,
                     out_space, ticket_out);
}

}  // extern "C"
