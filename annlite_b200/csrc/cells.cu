// cells.cu -- multi-cell (IVF) search over a set of existing handles: CellContainer.ivf_search
// (annlite/container.py:88-144) with the probe order of AnnLite._cell_selection (annlite/index.py:458-466).
//
//   cell_probe_kernel : one warp per query, the query's distance to every VQ centroid with annlite.math.cdist's formula
//                       for the metric (math.py:17-74, fp32), cells sorted by (distance, cell).
//   hnsw_walk4<8, EPL, true> (walk_fused.cu): the query's table is built once and walked over each probed cell.
//   ivf_merge_kernel  : one warp per query, the by-cell results read in probe order, the skip rule applied, the
//                       `limit` smallest kept by (distance, concatenation position).
#include <math_constants.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "annb_internal.h"

struct annb_cellset {
  std::vector<annb_index *> cells;
  int n_cells = 0, metric = 0, dim = 0, device = 0;
  annb_index *h0 = nullptr;         // its stream and scratch serve the cell set's launches
  float *d_centroids = nullptr;     // (n_cells, dim) or nullptr (then every search needs an explicit order)
  GraphDev *d_graphs = nullptr;     // (n_cells) descriptors, re-read before every fused search
  void *buf[8] = {nullptr};
  size_t cap[8] = {0};
  float probe_ms = 0, walk_ms = 0, merge_ms = 0;
  cudaEvent_t ev[6] = {nullptr};
  int last_route = 0;
};

namespace {

enum { C_QUERIES = 0, C_ORDER, C_K, C_LABELS, C_DISTS, C_FOUND, C_STATS, C_OUT };

int cs_buf(annb_cellset *cs, int slot, size_t bytes, void **out) {
  if (bytes == 0) bytes = 16;
  if (cs->cap[slot] < bytes) {
    if (cs->buf[slot]) {
      ANNB_CUDA(cudaStreamSynchronize(cs->h0->stream));
      ANNB_CUDA(cudaFree(cs->buf[slot]));
      cs->buf[slot] = nullptr;
      cs->cap[slot] = 0;
    }
    const size_t c = (bytes + bytes / 4 + 255) / 256 * 256;
    if (cudaMalloc(&cs->buf[slot], c) != cudaSuccess) {
      cudaGetLastError();
      ANNB_FAIL(ANNB_ENOMEM, "cudaMalloc(%zu bytes) failed", c);
    }
    cs->cap[slot] = c;
  }
  *out = cs->buf[slot];
  return ANNB_OK;
}

constexpr int PROBE_WARPS = 4;

// annlite.math.euclidean (math.py:57-74): sqrt(|y|^2 + |x|^2 - 2 x.y); cosine (:27-47):
// 1 - clip((x.y + eps) / (|x| |y| + eps), -1, 1).  fp32 like the reference's arrays; its sums run through numpy /
// BLAS, whose order this does not reproduce, so near-ties may order differently (a mismatch rate, like PQ encode).
// NaN (a negative rounding residue under the sqrt) sorts last, as numpy's argsort puts it.
__global__ void cell_probe_kernel(const float *__restrict__ x, const float *__restrict__ cen, int64_t B, int n_cells, int D,
                                  int cosine, int n_probe, int32_t *__restrict__ order) {
  __shared__ float sd[PROBE_WARPS][ANNB_MAX_CELLS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t q = (int64_t)blockIdx.x * PROBE_WARPS + warp;
  if (q >= B) return;
  const float *xq = x + q * D;
  float xx = 0.f;
  for (int j = lane; j < D; j += 32) xx = __fmaf_rn(xq[j], xq[j], xx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) xx += __shfl_xor_sync(0xffffffffu, xx, o);
  for (int c = lane; c < n_cells; c += 32) {
    const float *y = cen + (int64_t)c * D;
    float yy = 0.f, xy = 0.f;
    for (int j = 0; j < D; j++) {
      yy = __fmaf_rn(y[j], y[j], yy);
      xy = __fmaf_rn(xq[j], y[j], xy);
    }
    float d;
    if (cosine) {
      const float eps = 1.1920929e-07f;
      const float r = (xy + eps) / (sqrtf(xx) * sqrtf(yy) + eps);
      d = 1.f - fminf(fmaxf(r, -1.f), 1.f);
    } else {
      d = sqrtf(yy + xx - 2.f * xy);
    }
    sd[warp][c] = isnan(d) ? CUDART_INF_F : d;
  }
  __syncwarp();
  for (int c = lane; c < n_cells; c += 32) {
    const float d = sd[warp][c];
    int rank = 0;
    for (int j = 0; j < n_cells; j++) {
      const float e = sd[warp][j];
      rank += (e < d) || (e == d && j < c);
    }
    if (rank < n_probe) order[q * n_probe + rank] = c;
  }
}

constexpr int MERGE_WARPS = 4;

// CellContainer.ivf_search's loop and merge (container.py:101-138) for one query per warp.  Cell c's results are the
// first counts[q, c] entries of row (q, c) of the by-cell scratch, up to the first UINT64_MAX label; distances are
// taken as the per-cell searches return them to the container (`sqrt_in`: the raw walk distances, the EUCLIDEAN
// sqrt of HnswIndex.search applied here, hnsw/index.py:164-165).  In probe order a cell with no results is skipped
// (:104-105, :113-114), and a cell is dropped when `count >= limit` and its nearest distance is greater than the
// last appended cell's largest (:122-123).  The kept lists are concatenated and the `limit` smallest returned by
// (distance, concatenation position) -- the stable form of argsort(axis=0)[:limit] (:135); missing slots are
// +inf / UINT64_MAX / cell -1.
__global__ void ivf_merge_kernel(const float *__restrict__ sd, const uint64_t *__restrict__ sl, const int32_t *__restrict__ counts,
                                 const int32_t *__restrict__ order, int64_t B, int n_cells, int n_probe, int stride, int limit,
                                 int sqrt_in, float *__restrict__ od, uint64_t *__restrict__ ol, int32_t *__restrict__ oc) {
  __shared__ int app_cell[MERGE_WARPS][ANNB_MAX_CELLS], app_n[MERGE_WARPS][ANNB_MAX_CELLS];
  __shared__ int app_count[MERGE_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t q = (int64_t)blockIdx.x * MERGE_WARPS + warp;
  if (q >= B) return;
  auto dist = [&](int c, int i) {
    const float d = sd[(q * n_cells + c) * (int64_t)stride + i];
    return sqrt_in ? sqrtf(d) : d;
  };
  if (lane == 0) {
    int n_app = 0, count = 0;
    float tail = 0.f;
    for (int ci = 0; ci < n_probe; ci++) {
      const int c = order[q * n_probe + ci];
      const uint64_t *lab = sl + (q * n_cells + c) * (int64_t)stride;
      int n = min(counts[q * n_cells + c], stride);
      int v = 0;
      while (v < n && lab[v] != UINT64_MAX) v++;
      if (v == 0) continue;
      if (count >= limit && dist(c, 0) > tail) continue;
      app_cell[warp][n_app] = c;
      app_n[warp][n_app] = v;
      n_app++;
      count += v;
      tail = dist(c, v - 1);
    }
    app_count[warp] = n_app;
  }
  __syncwarp();
  const int n_app = app_count[warp];
  int total = 0;
  for (int a = 0; a < n_app; a++) {
    const int ca = app_cell[warp][a], na = app_n[warp][a];
    total += na;
    for (int i = lane; i < na; i += 32) {
      const float dx = dist(ca, i);
      int rank = i;
      for (int b = 0; b < n_app; b++) {
        if (b == a) continue;
        const int cb = app_cell[warp][b];
        int lo = 0, hi = app_n[warp][b];
        while (lo < hi) {  // entries of list b that precede (dx, position): <= before a, < after a
          const int mid = (lo + hi) >> 1;
          const float dm = dist(cb, mid);
          if (dm < dx || (b < a && dm == dx)) lo = mid + 1;
          else hi = mid;
        }
        rank += lo;
      }
      if (rank < limit) {
        od[q * limit + rank] = dx;
        ol[q * limit + rank] = sl[(q * n_cells + ca) * (int64_t)stride + i];
        oc[q * limit + rank] = ca;
      }
    }
  }
  for (int p = total + lane; p < limit; p += 32) {
    od[q * limit + p] = CUDART_INF_F;
    ol[q * limit + p] = UINT64_MAX;
    oc[q * limit + p] = -1;
  }
}

int launch_cell_probe(annb_cellset *cs, const float *dq, int64_t B, int n_probe, int32_t *d_order) {
  if (B == 0) return ANNB_OK;
  cell_probe_kernel<<<(unsigned)((B + PROBE_WARPS - 1) / PROBE_WARPS), PROBE_WARPS * 32, 0, cs->h0->stream>>>(
      dq, cs->d_centroids, B, cs->n_cells, cs->dim, cs->metric == ANNB_METRIC_COSINE, n_probe, d_order);
  cs->h0->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_ivf_merge(annb_cellset *cs, const float *sd, const uint64_t *sl, const int32_t *counts, const int32_t *order, int64_t B,
                     int n_probe, int stride, int limit, int sqrt_in, float *od, uint64_t *ol, int32_t *oc) {
  if (B == 0) return ANNB_OK;
  ivf_merge_kernel<<<(unsigned)((B + MERGE_WARPS - 1) / MERGE_WARPS), MERGE_WARPS * 32, 0, cs->h0->stream>>>(
      sd, sl, counts, order, B, cs->n_cells, n_probe, stride, limit, sqrt_in, od, ol, oc);
  cs->h0->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

// host or device input -> device pointer (cell-set buffer `slot` when it has to be copied)
int cs_stage(annb_cellset *cs, const void *p, int space, size_t bytes, int slot, const void **out) {
  if (space == ANNB_DEVICE) {
    *out = p;
    return ANNB_OK;
  }
  void *d;
  ANNB_TRY_RC(cs_buf(cs, slot, bytes, &d));
  ANNB_CUDA(cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, cs->h0->stream));
  *out = d;
  return ANNB_OK;
}

int check_order(const int32_t *order, int64_t B, int n_probe, int n_cells) {
  for (int64_t q = 0; q < B; q++)
    for (int i = 0; i < n_probe; i++) {
      const int32_t c = order[q * n_probe + i];
      if (c < 0 || c >= n_cells) ANNB_FAIL(ANNB_EINVAL, "probe order entry %d of query %lld is not a cell", c, (long long)q);
      for (int j = 0; j < i; j++)
        if (order[q * n_probe + j] == c) ANNB_FAIL(ANNB_EINVAL, "query %lld probes cell %d twice", (long long)q, c);
    }
  return ANNB_OK;
}

}  // namespace

extern "C" {

int annb_cellset_create(annb_index_t *const *handles, int n_cells, const float *centroids, int metric, annb_cellset_t **out) {
  if (!out || !handles) ANNB_FAIL(ANNB_EINVAL, "null argument");
  *out = nullptr;
  if (n_cells < 1 || n_cells > ANNB_MAX_CELLS) ANNB_FAIL(ANNB_ELIMIT, "n_cells=%d outside 1..ANNB_MAX_CELLS=%d", n_cells, ANNB_MAX_CELLS);
  if (metric == ANNB_METRIC_IP && centroids)
    ANNB_FAIL(ANNB_EINVAL, "cell selection has no inner-product distance (annlite.math.cdist knows cosine and euclidean)");
  annb_index *h0 = handles[0];
  for (int c = 0; c < n_cells; c++) {
    annb_index *h = handles[c];
    if (!h) ANNB_FAIL(ANNB_EINVAL, "cell %d: null handle", c);
    for (int j = 0; j < c; j++)
      if (handles[j] == h) ANNB_FAIL(ANNB_EINVAL, "cell %d repeats the handle of cell %d", c, j);
    if (h->device < 0) ANNB_FAIL(ANNB_ENODEVICE, "cell %d: host-only handle; a cell set searches on the GPU", c);
    if (h->device != h0->device) ANNB_FAIL(ANNB_EINVAL, "cell %d is on device %d, cell 0 on device %d", c, h->device, h0->device);
    if (h->metric != h0->metric || h->dim != h0->dim || h->M != h0->M || h->Ks != h0->Ks)
      ANNB_FAIL(ANNB_EINVAL, "cell %d: metric / dim / PQ geometry differ from cell 0", c);
    if (h->h_codebook.empty()) ANNB_FAIL(ANNB_ESTATE, "cell %d: no PQ codebook set", c);
    if (h->h_codebook != h0->h_codebook) ANNB_FAIL(ANNB_EINVAL, "cell %d: its PQ codebook differs from cell 0's (the cells share one codec)", c);
  }
  if (centroids && metric != h0->metric) ANNB_FAIL(ANNB_EINVAL, "metric %d differs from the cells' metric %d", metric, h0->metric);
  ANNB_CUDA(cudaSetDevice(h0->device));
  annb_cellset *cs = new annb_cellset();
  cs->cells.assign(handles, handles + n_cells);
  cs->n_cells = n_cells;
  cs->metric = h0->metric;
  cs->dim = h0->dim;
  cs->h0 = h0;
  cs->device = h0->device;
  cudaError_t e = cudaMalloc(&cs->d_graphs, sizeof(GraphDev) * n_cells);
  if (e == cudaSuccess && centroids) {
    e = cudaMalloc(&cs->d_centroids, sizeof(float) * n_cells * cs->dim);
    if (e == cudaSuccess) e = cudaMemcpy(cs->d_centroids, centroids, sizeof(float) * n_cells * cs->dim, cudaMemcpyHostToDevice);
  }
  for (int i = 0; i < 6 && e == cudaSuccess; i++) e = cudaEventCreate(&cs->ev[i]);
  if (e != cudaSuccess) {
    annb_set_error("CUDA error %s while creating a cell set", cudaGetErrorString(e));
    annb_cellset_destroy(cs);
    return ANNB_ECUDA;
  }
  *out = cs;
  return ANNB_OK;
}

int annb_cellset_destroy(annb_cellset_t *cs) {
  if (!cs) return ANNB_OK;
  // the handles may be gone already (a cell set only borrows them): cudaFree waits for the work using the buffers
  cudaSetDevice(cs->device);
  for (void *p : cs->buf)
    if (p) cudaFree(p);
  if (cs->d_graphs) cudaFree(cs->d_graphs);
  if (cs->d_centroids) cudaFree(cs->d_centroids);
  for (cudaEvent_t e : cs->ev)
    if (e) cudaEventDestroy(e);
  delete cs;
  return ANNB_OK;
}

int annb_cellset_search(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int normalize,
                        const int32_t *order, int n_probe, int limit, int ef, int flags, uint64_t *labels_out,
                        float *dists_out, int32_t *cells_out, int out_space, uint64_t *part_labels, float *part_dists,
                        int64_t *part_stats) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  const int C = cs->n_cells;
  if (B < 0 || limit <= 0 || ef <= 0 || !labels_out || !dists_out || !cells_out || (B > 0 && !queries))
    ANNB_FAIL(ANNB_EINVAL, "bad B / limit / ef / outputs");
  if (n_probe < 1 || n_probe > C) ANNB_FAIL(ANNB_EINVAL, "n_probe=%d outside 1..n_cells=%d", n_probe, C);
  if (!order && !cs->d_centroids) ANNB_FAIL(ANNB_ESTATE, "no centroids: pass the probe order");
  if (std::max(ef, limit) > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "max(ef, limit)=%d exceeds ANNB_MAX_EF=%d", std::max(ef, limit), ANNB_MAX_EF);
  if (order && in_space != ANNB_DEVICE) ANNB_TRY_RC(check_order(order, B, n_probe, C));
  annb_index *h0 = cs->h0;
  ANNB_CUDA(cudaSetDevice(h0->device));
  // every cell's device graph up to date and its descriptor read now: buffers move on resize, nothing is cached
  std::vector<GraphDev> gd(C);
  std::vector<int32_t> kc(C);
  bool fused = !(flags & ANNB_CELLS_GENERIC);
  for (int c = 0; c < C; c++) {
    annb_index *h = cs->cells[c];
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "cell %d: index not initialised", c);
    ANNB_TRY_RC(sync_device_graph(h));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream2));
    gd[c] = h->gd;
    const int64_t live = h->g.count.load() - h->g.num_deleted;
    kc[c] = (int32_t)std::min<int64_t>(limit, std::max<int64_t>(live, 0));  // container.py:104-105, :119
    fused &= h->g.num_deleted == 0 && !h->opt_force_general && walk4_can_fuse(h) && h->M == 8;
  }
  cs->last_route = fused ? 0 : 1;
  if (B == 0) return ANNB_OK;
  cudaStream_t st = h0->stream;
  const bool host_out = out_space != ANNB_DEVICE;
  // staged queries: the probe reads them raw, the walk normalised
  float *dq;
  const size_t qbytes = (size_t)B * cs->dim * sizeof(float);
  ANNB_TRY_RC(cs_buf(cs, C_QUERIES, qbytes, (void **)&dq));
  ANNB_CUDA(cudaMemcpyAsync(dq, queries, qbytes, in_space == ANNB_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  int32_t *dorder;
  if (order) {
    ANNB_TRY_RC(cs_stage(cs, order, in_space, (size_t)B * n_probe * 4, C_ORDER, (const void **)&dorder));
  } else {
    ANNB_TRY_RC(cs_buf(cs, C_ORDER, (size_t)B * n_probe * 4, (void **)&dorder));
    cudaEventRecord(cs->ev[0], st);
    ANNB_TRY_RC(launch_cell_probe(cs, dq, B, n_probe, dorder));
    cudaEventRecord(cs->ev[1], st);
  }
  // by-cell scratch (B, n_cells, limit)
  const size_t slots = (size_t)B * C;
  uint64_t *sl;
  float *sd;
  int32_t *sfound;
  int64_t *sstats = nullptr;
  ANNB_TRY_RC(cs_buf(cs, C_LABELS, slots * limit * 8, (void **)&sl));
  ANNB_TRY_RC(cs_buf(cs, C_DISTS, slots * limit * 4, (void **)&sd));
  ANNB_TRY_RC(cs_buf(cs, C_FOUND, slots * 4, (void **)&sfound));
  if (part_stats) ANNB_TRY_RC(cs_buf(cs, C_STATS, slots * 24, (void **)&sstats));
  ANNB_CUDA(cudaMemsetAsync(sl, 0xff, slots * limit * 8, st));  // cells a query does not probe stay empty
  ANNB_CUDA(cudaMemsetAsync(sfound, 0, slots * 4, st));
  if (sstats) ANNB_CUDA(cudaMemsetAsync(sstats, 0, slots * 24, st));
  if (fused) {
    for (int r = 0; r < normalize; r++) ANNB_TRY_RC(launch_l2_normalize(h0, dq, B, cs->dim));
    int32_t *dk;
    ANNB_TRY_RC(cs_buf(cs, C_K, (size_t)C * 4, (void **)&dk));
    ANNB_CUDA(cudaMemcpyAsync(cs->d_graphs, gd.data(), sizeof(GraphDev) * C, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dk, kc.data(), (size_t)C * 4, cudaMemcpyHostToDevice, st));
    SearchParams p;
    memset(&p, 0, sizeof(p));
    p.queries = dq;
    p.cbt = h0->d_codebook_t;
    p.cb_vec = h0->cb_vec;
    p.ds = h0->ds;
    p.is_ip = h0->metric != ANNB_METRIC_L2;
    p.bias = h0->opt_ip_raw ? 0.f : (float)(1.0 / (double)h0->Ks);
    p.B = B;
    p.k = limit;
    p.ef = ef;
    p.out_labels = sl;
    p.out_dists = sd;
    p.out_found = sfound;
    p.out_stats = sstats;
    p.cells = cs->d_graphs;
    p.cell_order = dorder;
    p.cell_k = dk;
    p.n_cells = C;
    p.n_probe = n_probe;
    p.cell_limit = limit;  // row length of the scratch; every k_c <= limit
    std::lock_guard<std::mutex> lk(h0->mu);
    cudaEventRecord(cs->ev[2], st);
    const int rc = launch_walk4_cells(h0, p);
    if (rc == 1) ANNB_FAIL(ANNB_ESTATE, "the multi-cell walk does not apply to these cells");
    if (rc) return rc;
    cudaEventRecord(cs->ev[3], st);
  } else {
    // generic route: one annb_search per probed cell over the whole batch (deletion-aware, any geometry), its
    // outputs copied into the cell's slot of the scratch
    std::vector<char> probed(C, 0);
    if (order && in_space != ANNB_DEVICE) {
      for (int64_t i = 0; i < B * n_probe; i++) probed[order[i]] = 1;
    } else {
      std::vector<int32_t> ho((size_t)B * n_probe);
      ANNB_CUDA(cudaMemcpyAsync(ho.data(), dorder, ho.size() * 4, cudaMemcpyDeviceToHost, st));
      ANNB_CUDA(cudaStreamSynchronize(st));
      for (int32_t c : ho) probed[c] = 1;
    }
    ANNB_CUDA(cudaStreamSynchronize(st));
    cudaEventRecord(cs->ev[2], st);
    std::vector<uint64_t> hl;
    std::vector<float> hd;
    std::vector<int64_t> hs(part_stats ? (size_t)B * 3 : 0);
    std::vector<int32_t> hk((size_t)B);
    for (int c = 0; c < C; c++) {
      if (!probed[c] || kc[c] == 0) continue;
      const int k = kc[c];
      hl.resize((size_t)B * k);
      hd.resize((size_t)B * k);
      const int rc = annb_search(cs->cells[c], queries, nullptr, in_space, B, normalize, k, ef, nullptr, ANNB_HOST, 0, hl.data(),
                                 hd.data(), ANNB_HOST, part_stats ? hs.data() : nullptr);
      if (rc && rc != ANNB_EFEWRESULTS) return rc;  // a short row is padded with UINT64_MAX: the merge stops there
      std::fill(hk.begin(), hk.end(), k);
      ANNB_CUDA(cudaMemcpy2DAsync(sl + (size_t)c * limit, (size_t)C * limit * 8, hl.data(), (size_t)k * 8, (size_t)k * 8, (size_t)B,
                                  cudaMemcpyHostToDevice, st));
      ANNB_CUDA(cudaMemcpy2DAsync(sd + (size_t)c * limit, (size_t)C * limit * 4, hd.data(), (size_t)k * 4, (size_t)k * 4, (size_t)B,
                                  cudaMemcpyHostToDevice, st));
      ANNB_CUDA(cudaMemcpy2DAsync(sfound + c, (size_t)C * 4, hk.data(), 4, 4, (size_t)B, cudaMemcpyHostToDevice, st));
      if (part_stats)
        ANNB_CUDA(cudaMemcpy2DAsync(sstats + (size_t)c * 3, (size_t)C * 24, hs.data(), 24, 24, (size_t)B, cudaMemcpyHostToDevice, st));
      ANNB_CUDA(cudaStreamSynchronize(st));  // the host buffers are reused by the next cell
    }
    cudaEventRecord(cs->ev[3], st);
  }
  // merge
  uint64_t *ol = labels_out;
  float *od = dists_out;
  int32_t *oc = cells_out;
  if (host_out) {
    void *o;
    ANNB_TRY_RC(cs_buf(cs, C_OUT, (size_t)B * limit * 16, &o));
    ol = (uint64_t *)o;
    od = reinterpret_cast<float *>(ol + (size_t)B * limit);
    oc = reinterpret_cast<int32_t *>(od + (size_t)B * limit);
  }
  cudaEventRecord(cs->ev[4], st);
  ANNB_TRY_RC(launch_ivf_merge(cs, sd, sl, sfound, dorder, B, n_probe, limit, limit, cs->metric == ANNB_METRIC_L2, od, ol, oc));
  cudaEventRecord(cs->ev[5], st);
  if (host_out) {
    ANNB_CUDA(cudaMemcpyAsync(labels_out, ol, (size_t)B * limit * 8, cudaMemcpyDeviceToHost, st));
    ANNB_CUDA(cudaMemcpyAsync(dists_out, od, (size_t)B * limit * 4, cudaMemcpyDeviceToHost, st));
    ANNB_CUDA(cudaMemcpyAsync(cells_out, oc, (size_t)B * limit * 4, cudaMemcpyDeviceToHost, st));
  }
  const cudaMemcpyKind dh = host_out ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  if (part_labels) ANNB_CUDA(cudaMemcpyAsync(part_labels, sl, slots * limit * 8, dh, st));
  if (part_dists) ANNB_CUDA(cudaMemcpyAsync(part_dists, sd, slots * limit * 4, dh, st));
  if (part_stats) ANNB_CUDA(cudaMemcpyAsync(part_stats, sstats, slots * 24, dh, st));
  ANNB_CUDA(cudaStreamSynchronize(st));
  if (h0->opt_timing) {
    cs->probe_ms = 0;
    if (!order) cudaEventElapsedTime(&cs->probe_ms, cs->ev[0], cs->ev[1]);
    cudaEventElapsedTime(&cs->walk_ms, cs->ev[2], cs->ev[3]);
    cudaEventElapsedTime(&cs->merge_ms, cs->ev[4], cs->ev[5]);
  }
  return ANNB_OK;
}

int annb_cellset_merge(annb_cellset_t *cs, const uint64_t *labels, const float *dists, const int32_t *counts,
                       const int32_t *order, int in_space, int64_t B, int n_probe, int limit, uint64_t *labels_out,
                       float *dists_out, int32_t *cells_out, int out_space) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  const int C = cs->n_cells;
  if (B < 0 || limit <= 0 || !labels || !dists || !counts || !order || !labels_out || !dists_out || !cells_out)
    ANNB_FAIL(ANNB_EINVAL, "bad B / limit / buffers");
  if (n_probe < 1 || n_probe > C) ANNB_FAIL(ANNB_EINVAL, "n_probe=%d outside 1..n_cells=%d", n_probe, C);
  if (in_space != ANNB_DEVICE) ANNB_TRY_RC(check_order(order, B, n_probe, C));
  if (B == 0) return ANNB_OK;
  ANNB_CUDA(cudaSetDevice(cs->h0->device));
  const size_t slots = (size_t)B * C;
  const void *dl, *dd, *dc, *dor;
  ANNB_TRY_RC(cs_stage(cs, labels, in_space, slots * limit * 8, C_LABELS, &dl));
  ANNB_TRY_RC(cs_stage(cs, dists, in_space, slots * limit * 4, C_DISTS, &dd));
  ANNB_TRY_RC(cs_stage(cs, counts, in_space, slots * 4, C_FOUND, &dc));
  ANNB_TRY_RC(cs_stage(cs, order, in_space, (size_t)B * n_probe * 4, C_ORDER, &dor));
  const bool host_out = out_space != ANNB_DEVICE;
  uint64_t *ol = labels_out;
  float *od = dists_out;
  int32_t *oc = cells_out;
  if (host_out) {
    void *o;
    ANNB_TRY_RC(cs_buf(cs, C_OUT, (size_t)B * limit * 16, &o));
    ol = (uint64_t *)o;
    od = reinterpret_cast<float *>(ol + (size_t)B * limit);
    oc = reinterpret_cast<int32_t *>(od + (size_t)B * limit);
  }
  cudaStream_t st = cs->h0->stream;
  cudaEventRecord(cs->ev[4], st);
  ANNB_TRY_RC(launch_ivf_merge(cs, (const float *)dd, (const uint64_t *)dl, (const int32_t *)dc, (const int32_t *)dor, B, n_probe,
                               limit, limit, 0, od, ol, oc));
  cudaEventRecord(cs->ev[5], st);
  if (host_out) {
    ANNB_CUDA(cudaMemcpyAsync(labels_out, ol, (size_t)B * limit * 8, cudaMemcpyDeviceToHost, st));
    ANNB_CUDA(cudaMemcpyAsync(dists_out, od, (size_t)B * limit * 4, cudaMemcpyDeviceToHost, st));
    ANNB_CUDA(cudaMemcpyAsync(cells_out, oc, (size_t)B * limit * 4, cudaMemcpyDeviceToHost, st));
  }
  ANNB_CUDA(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&cs->merge_ms, cs->ev[4], cs->ev[5]);
  return ANNB_OK;
}

int annb_cellset_probe(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int n_probe, int32_t *order_out,
                       int out_space) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (!cs->d_centroids) ANNB_FAIL(ANNB_ESTATE, "the cell set has no centroids");
  if (n_probe < 1 || n_probe > cs->n_cells) ANNB_FAIL(ANNB_EINVAL, "n_probe=%d outside 1..n_cells=%d", n_probe, cs->n_cells);
  if (B < 0 || (B > 0 && (!queries || !order_out))) ANNB_FAIL(ANNB_EINVAL, "bad B / buffers");
  if (B == 0) return ANNB_OK;
  ANNB_CUDA(cudaSetDevice(cs->h0->device));
  const float *dq;
  ANNB_TRY_RC(cs_stage(cs, queries, in_space, (size_t)B * cs->dim * 4, C_QUERIES, (const void **)&dq));
  int32_t *o = order_out;
  if (out_space != ANNB_DEVICE) ANNB_TRY_RC(cs_buf(cs, C_ORDER, (size_t)B * n_probe * 4, (void **)&o));
  cudaStream_t st = cs->h0->stream;
  cudaEventRecord(cs->ev[0], st);
  ANNB_TRY_RC(launch_cell_probe(cs, dq, B, n_probe, o));
  cudaEventRecord(cs->ev[1], st);
  if (out_space != ANNB_DEVICE) ANNB_CUDA(cudaMemcpyAsync(order_out, o, (size_t)B * n_probe * 4, cudaMemcpyDeviceToHost, st));
  ANNB_CUDA(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&cs->probe_ms, cs->ev[0], cs->ev[1]);
  return ANNB_OK;
}

int annb_cellset_last_ms(annb_cellset_t *cs, float *probe_ms, float *walk_ms, float *merge_ms, int *route) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (probe_ms) *probe_ms = cs->probe_ms;
  if (walk_ms) *walk_ms = cs->walk_ms;
  if (merge_ms) *merge_ms = cs->merge_ms;
  if (route) *route = cs->last_route;
  return ANNB_OK;
}

}  // extern "C"
