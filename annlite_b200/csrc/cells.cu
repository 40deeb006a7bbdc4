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
#include <map>
#include <vector>

#include "annb_internal.h"

struct annb_cellset {
  std::vector<annb_index *> cells;
  int n_cells = 0, metric = 0, dim = 0, device = 0;
  annb_index *h0 = nullptr;         // its stream and scratch serve the cell set's launches
  float *d_centroids = nullptr;     // (n_cells, dim) or nullptr (then every search needs an explicit order)
  GraphDev *d_graphs = nullptr;     // (n_cells) descriptors, re-read before every fused search
  void *buf[26] = {nullptr};
  size_t cap[26] = {0};
  float probe_ms = 0, walk_ms = 0, merge_ms = 0;
  cudaEvent_t ev[8] = {nullptr};    // [0,1] probe, [2,3] walk, [4,5] merge, [6,7] hand-over to a cell's stream and back
  int last_route = 0;
  int64_t last_rerun_pairs = 0;     // annb_cellset_search_prepared / _multi: (query, cell) pairs re-run on the bitmap walk
  int last_handle_cells = 0;        // ... and cells served by their own filtered launch instead of the fused walk
  std::vector<int64_t> below;       // annb_cellset_set_bruteforce: per cell, scan filters admitting <= this many (-1 = never)
  int64_t last_scanned_pairs = 0;   // (query, cell) pairs the last search scanned exactly ...
  int64_t last_scanned_rows = 0;    // ... and the rows those scans scored
  CellBuildStats build;             // annb_cellset_add_items: the last call's one-pass build ...
  int build_cells = 0;              // ... and the cells it served
};

namespace {

enum { C_QUERIES = 0, C_ORDER, C_K, C_LABELS, C_DISTS, C_FOUND, C_STATS, C_OUT, C_BITS, C_TABLES, C_TMP_L, C_TMP_D, C_TMP_F,
       C_TMP_S, C_QMAP, C_SLOT, C_SLOT_K, C_SLOT_BITS, C_GTABLES, C_QF, C_SCAN_JOBS, C_SCAN_ROWS, C_SCAN_QUERIES,
       C_SCAN_BLOCKS, C_SCAN_PARTS, C_SCAN_DONE };
static_assert(C_SCAN_DONE < 26, "annb_cellset::buf is too small");

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

// a batch staged for a cell-set search: queries (raw; the walk normalises them in place), probe order, and the by-cell
// scratch (B, n_cells, limit), emptied
struct Staged {
  float *dq = nullptr;
  int32_t *dorder = nullptr;
  uint64_t *sl = nullptr;
  float *sd = nullptr;
  int32_t *sfound = nullptr;
  int64_t *sstats = nullptr;
  float *tables = nullptr;  // the K1 tables of the whole batch once batch_tables has built them
};

int stage_batch(annb_cellset *cs, const float *queries, int in_space, int64_t B, const int32_t *order, int n_probe, int limit,
                bool stats, Staged &b) {
  cudaStream_t st = cs->h0->stream;
  // staged queries: the probe reads them raw, the walk normalised
  const size_t qbytes = (size_t)B * cs->dim * sizeof(float);
  ANNB_TRY_RC(cs_buf(cs, C_QUERIES, qbytes, (void **)&b.dq));
  ANNB_CUDA(cudaMemcpyAsync(b.dq, queries, qbytes, in_space == ANNB_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  if (order) {
    ANNB_TRY_RC(cs_stage(cs, order, in_space, (size_t)B * n_probe * 4, C_ORDER, (const void **)&b.dorder));
  } else {
    ANNB_TRY_RC(cs_buf(cs, C_ORDER, (size_t)B * n_probe * 4, (void **)&b.dorder));
    cudaEventRecord(cs->ev[0], st);
    ANNB_TRY_RC(launch_cell_probe(cs, b.dq, B, n_probe, b.dorder));
    cudaEventRecord(cs->ev[1], st);
  }
  // by-cell scratch (B, n_cells, limit)
  const size_t slots = (size_t)B * cs->n_cells;
  ANNB_TRY_RC(cs_buf(cs, C_LABELS, slots * limit * 8, (void **)&b.sl));
  ANNB_TRY_RC(cs_buf(cs, C_DISTS, slots * limit * 4, (void **)&b.sd));
  ANNB_TRY_RC(cs_buf(cs, C_FOUND, slots * 4, (void **)&b.sfound));
  if (stats) ANNB_TRY_RC(cs_buf(cs, C_STATS, slots * 24, (void **)&b.sstats));
  ANNB_CUDA(cudaMemsetAsync(b.sl, 0xff, slots * limit * 8, st));  // cells a query does not probe stay empty
  ANNB_CUDA(cudaMemsetAsync(b.sfound, 0, slots * 4, st));
  if (b.sstats) ANNB_CUDA(cudaMemsetAsync(b.sstats, 0, slots * 24, st));
  return ANNB_OK;
}

// the parameters of a multi-cell walk over a staged batch (fused table build from the normalised queries)
void cells_params(annb_cellset *cs, const Staged &b, int64_t B, int n_probe, int limit, int ef, const int32_t *dk, SearchParams &p) {
  const annb_index *h0 = cs->h0;
  memset(&p, 0, sizeof(p));
  p.queries = b.dq;
  p.cbt = h0->d_codebook_t;
  p.cb_vec = h0->cb_vec;
  p.ds = h0->ds;
  p.is_ip = h0->metric != ANNB_METRIC_L2;
  p.bias = h0->opt_ip_raw ? 0.f : (float)(1.0 / (double)h0->Ks);
  p.B = B;
  p.k = limit;
  p.ef = ef;
  p.out_labels = b.sl;
  p.out_dists = b.sd;
  p.out_found = b.sfound;
  p.out_stats = b.sstats;
  p.cells = cs->d_graphs;
  p.cell_order = b.dorder;
  p.cell_k = dk;
  p.n_cells = cs->n_cells;
  p.n_probe = n_probe;
  p.cell_limit = limit;  // row length of the scratch; every k_c <= limit
}

// the probe order on the host: the caller's, or a copy of the device one
int host_order(annb_cellset *cs, const int32_t *order, int in_space, const int32_t *dorder, int64_t B, int n_probe,
               std::vector<int32_t> &tmp, const int32_t **out) {
  if (order && in_space != ANNB_DEVICE) {
    *out = order;
    return ANNB_OK;
  }
  tmp.resize((size_t)B * n_probe);
  ANNB_CUDA(cudaMemcpyAsync(tmp.data(), dorder, tmp.size() * 4, cudaMemcpyDeviceToHost, cs->h0->stream));
  ANNB_CUDA(cudaStreamSynchronize(cs->h0->stream));
  *out = tmp.data();
  return ANNB_OK;
}

// rows of one cell's (B, k) search outputs -> that cell's rows (q * n_cells + c) of the by-cell scratch: every row, or
// (idx) the rows a re-run wrote, idx[i] = query row; `dense` = the outputs hold only those rows, row i for query idx[i]
__global__ void cell_scatter_kernel(const uint64_t *__restrict__ il, const float *__restrict__ id, const int32_t *__restrict__ ifound,
                                    const int64_t *__restrict__ istats, const uint32_t *__restrict__ idx, int64_t n, int k,
                                    int n_cells, int c, int stride, int dense, uint64_t *__restrict__ sl, float *__restrict__ sd,
                                    int32_t *__restrict__ sfound, int64_t *__restrict__ sstats) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t i = t / k;
  if (i >= n) return;
  const int j = (int)(t - i * k);
  const int64_t q = idx ? (int64_t)idx[i] : i;
  const int64_t r = dense ? i : q;  // input row
  const int64_t o = q * n_cells + c;
  sl[o * stride + j] = il[r * k + j];
  sd[o * stride + j] = id[r * k + j];
  if (j == 0) {
    sfound[o] = ifound[r];
    if (sstats)
      for (int s = 0; s < 3; s++) sstats[o * 3 + s] = istats[r * 3 + s];
  }
}

int launch_cell_scatter(cudaStream_t st, const uint64_t *il, const float *id, const int32_t *ifound, const int64_t *istats,
                        const uint32_t *idx, int64_t n, int k, int n_cells, int c, int stride, uint64_t *sl, float *sd,
                        int32_t *sfound, int64_t *sstats, bool dense = false) {
  if (n == 0) return ANNB_OK;
  const int64_t total = n * k;
  cell_scatter_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(il, id, ifound, istats, idx, n, k, n_cells, c, stride,
                                                                        dense ? 1 : 0, sl, sd, sfound, sstats);
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

// Generic route: for every probed cell with k_c > 0, one search of the whole batch into host buffers
// (search(c, k, labels, dists, stats) -> status), copied into the cell's slot of the scratch.
template <class Search>
int per_cell_route(annb_cellset *cs, const int32_t *order, int in_space, const int32_t *dorder, int64_t B, int n_probe, int limit,
                   const std::vector<int32_t> &kc, uint64_t *sl, float *sd, int32_t *sfound, int64_t *sstats, Search search) {
  const int C = cs->n_cells;
  cudaStream_t st = cs->h0->stream;
  std::vector<char> probed(C, 0);
  std::vector<int32_t> tmp;
  const int32_t *ho;
  ANNB_TRY_RC(host_order(cs, order, in_space, dorder, B, n_probe, tmp, &ho));
  for (int64_t i = 0; i < B * n_probe; i++) probed[ho[i]] = 1;
  ANNB_CUDA(cudaStreamSynchronize(st));
  cudaEventRecord(cs->ev[2], st);
  std::vector<uint64_t> hl;
  std::vector<float> hd;
  std::vector<int64_t> hs(sstats ? (size_t)B * 3 : 0);
  std::vector<int32_t> hk((size_t)B);
  for (int c = 0; c < C; c++) {
    if (!probed[c] || kc[c] == 0) continue;
    const int k = kc[c];
    hl.resize((size_t)B * k);
    hd.resize((size_t)B * k);
    ANNB_TRY_RC(search(c, k, hl.data(), hd.data(), sstats ? hs.data() : nullptr));
    std::fill(hk.begin(), hk.end(), k);
    ANNB_CUDA(cudaMemcpy2DAsync(sl + (size_t)c * limit, (size_t)C * limit * 8, hl.data(), (size_t)k * 8, (size_t)k * 8, (size_t)B,
                                cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpy2DAsync(sd + (size_t)c * limit, (size_t)C * limit * 4, hd.data(), (size_t)k * 4, (size_t)k * 4, (size_t)B,
                                cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpy2DAsync(sfound + c, (size_t)C * 4, hk.data(), 4, 4, (size_t)B, cudaMemcpyHostToDevice, st));
    if (sstats)
      ANNB_CUDA(cudaMemcpy2DAsync(sstats + (size_t)c * 3, (size_t)C * 24, hs.data(), 24, 24, (size_t)B, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaStreamSynchronize(st));  // the host buffers are reused by the next cell
  }
  cudaEventRecord(cs->ev[3], st);
  return ANNB_OK;
}

// The merge over the by-cell scratch, the outputs and the parts copied out (out_space), one synchronisation, timings.
int merge_and_finish(annb_cellset *cs, const float *sd, const uint64_t *sl, const int32_t *sfound, const int64_t *sstats,
                     const int32_t *dorder, bool probed_here, int64_t B, int n_probe, int limit, uint64_t *labels_out,
                     float *dists_out, int32_t *cells_out, int out_space, uint64_t *part_labels, float *part_dists,
                     int64_t *part_stats) {
  cudaStream_t st = cs->h0->stream;
  const size_t slots = (size_t)B * cs->n_cells;
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
  if (cs->h0->opt_timing) {
    cs->probe_ms = 0;
    if (probed_here) cudaEventElapsedTime(&cs->probe_ms, cs->ev[0], cs->ev[1]);
    cudaEventElapsedTime(&cs->walk_ms, cs->ev[2], cs->ev[3]);
    cudaEventElapsedTime(&cs->merge_ms, cs->ev[4], cs->ev[5]);
  }
  return ANNB_OK;
}

// One exact subset scan of a cell-set search: cell `cell`'s prepared filter `f` (its admitted rows in id order, or a
// label list's live entries in order), or with f == nullptr the cell's `live` rows in id order (`dead` = its deletion
// bitmap, nullptr when nothing is deleted), scanned for the query rows `rows` with k results each.
struct ScanPlan {
  int cell = 0, k = 0;
  const PreparedFilter *f = nullptr;
  int64_t live = 0;
  const uint32_t *dead = nullptr;
  std::vector<uint32_t> rows;
};

int64_t plan_rows(const ScanPlan &p) { return !p.f ? p.live : (p.f->ids ? p.f->n_ids : p.f->count); }

// a scanned pair with fewer live subset entries than its k fails as annb_scan_subset fails
int check_plans(const std::vector<ScanPlan> &plans) {
  for (const ScanPlan &p : plans)
    if (!p.rows.empty() && plan_rows(p) < p.k)
      ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
  return ANNB_OK;
}

// The scans of a search, uploaded: the job table, the query rows and tiles, and the launch groups
struct StagedScans {
  std::vector<SubsetScan> jobs;
  std::vector<std::pair<size_t, size_t>> groups;  // [first, last) jobs of each launch
  std::vector<int64_t> tile0;                     // first tile of each launch (+ the end)
  std::vector<SubsetChunks> chunks;               // each launch's row chunks
  std::vector<int64_t> tile_groups;               // ... and its (job, first query) tiles, whose counters it zeroes
  SubsetScan *djobs = nullptr;
  int4 *dtiles = nullptr;
};

// The plans (in cell order) staged on the cell set's stream, before the walk: one gather and one scan for all plans, or
// (per_cell) for each cell's plans in turn.  Counts the scanned pairs and rows.
int stage_scans(annb_cellset *cs, const std::vector<ScanPlan> &plans, const std::vector<const uint8_t *> &own,
                const std::vector<GraphDev> &gd, bool per_cell, StagedScans &ss) {
  const size_t J = plans.size();
  if (J == 0) return ANNB_OK;
  cudaStream_t st = cs->h0->stream;
  int64_t rows = 0, blocks = 0, nq = 0;
  for (const ScanPlan &p : plans) {
    const int64_t span = p.f ? p.f->n : gd[(size_t)p.cell].n;  // ids a bitmap covers
    if (p.f || p.dead) rows += plan_rows(p);                   // (a live-rows plan without deletions is scanned in place)
    if (p.f ? !p.f->ids : p.dead != nullptr) blocks += ((span + 31) / 32 + 255) / 256;
    nq += (int64_t)p.rows.size();
  }
  // launch groups: [g0, g1) ranges of plans, each with its tiles
  std::vector<std::pair<size_t, size_t>> &groups = ss.groups;
  for (size_t j = 0; j < J; j++)
    if (groups.empty() || (per_cell && plans[j].cell != plans[groups.back().first].cell)) groups.push_back({j, j + 1});
    else groups.back().second = j + 1;
  // tiles {job in the launch, first query, chunk, tile group}: a launch whose tiles are too few to fill the GPU cuts its
  // subsets into row chunks (subset_scan_chunk_rows); its chunk lists take (tile groups, width, G, K) entries
  std::vector<int4> tiles;
  std::vector<int64_t> &tile0 = ss.tile0;
  size_t part_entries = 0, max_groups = 0;
  for (auto &g : groups) {
    int kmax = 1;
    for (size_t j = g.first; j < g.second; j++) kmax = std::max(kmax, plans[j].k);
    const int w = subset_scan_tile_width(kmax);
    int64_t n_groups = 0, longest = 0;
    for (size_t j = g.first; j < g.second; j++) {
      n_groups += ((int64_t)plans[j].rows.size() + w - 1) / w;
      if (!plans[j].rows.empty()) longest = std::max(longest, plan_rows(plans[j]));
    }
    SubsetChunks ch;
    memset(&ch, 0, sizeof(ch));
    ch.rows = subset_scan_chunk_rows(cs->h0, n_groups, longest);
    ch.K = kmax;
    ch.G = ch.rows ? (int)((longest + ch.rows - 1) / ch.rows) : 1;
    tile0.push_back((int64_t)tiles.size());
    int group = 0;
    for (size_t j = g.first; j < g.second; j++) {
      const int nch = ch.rows ? (int)((plan_rows(plans[j]) + ch.rows - 1) / ch.rows) : 1;
      for (size_t q0 = 0; q0 < plans[j].rows.size(); q0 += (size_t)w, group++)
        for (int c = 0; c < nch; c++) tiles.push_back(make_int4((int)(j - g.first), (int)q0, c, group));
    }
    if (ch.rows) {
      part_entries = std::max(part_entries, (size_t)n_groups * w * ch.G * ch.K);
      max_groups = std::max(max_groups, (size_t)n_groups);
    }
    ss.chunks.push_back(ch);
    ss.tile_groups.push_back(n_groups);
  }
  tile0.push_back((int64_t)tiles.size());
  if (part_entries) {
    void *pp;
    unsigned int *done;
    ANNB_TRY_RC(cs_buf(cs, C_SCAN_PARTS, part_entries * 8, &pp));
    ANNB_TRY_RC(cs_buf(cs, C_SCAN_DONE, max_groups * 4, (void **)&done));
    for (SubsetChunks &ch : ss.chunks)
      if (ch.rows) {
        ch.part_d = (float *)pp;
        ch.part_i = reinterpret_cast<uint32_t *>((float *)pp + part_entries);
        ch.done = done;
      }
  }
  uint64_t *glab;
  uint32_t *dq;
  unsigned int *boffs;
  SubsetScan *djobs;
  const size_t qwords = ((size_t)nq + 3) / 4 * 4;  // the int4 tiles follow the query rows: 16-byte aligned
  ANNB_TRY_RC(cs_buf(cs, C_SCAN_ROWS, (size_t)rows * 16, (void **)&glab));
  ANNB_TRY_RC(cs_buf(cs, C_SCAN_QUERIES, qwords * 4 + tiles.size() * sizeof(int4), (void **)&dq));
  ANNB_TRY_RC(cs_buf(cs, C_SCAN_BLOCKS, (size_t)blocks * 4, (void **)&boffs));
  ANNB_TRY_RC(cs_buf(cs, C_SCAN_JOBS, J * sizeof(SubsetScan), (void **)&djobs));
  int4 *dtiles = reinterpret_cast<int4 *>(dq + qwords);
  uint8_t *gcodes = reinterpret_cast<uint8_t *>(glab + rows);
  std::vector<SubsetScan> &jobs = ss.jobs;
  jobs.resize(J);
  std::vector<uint32_t> hq;
  hq.reserve((size_t)nq);
  int64_t r0 = 0, bl0 = 0;
  for (size_t j = 0; j < J; j++) {
    const ScanPlan &p = plans[j];
    SubsetScan &s = jobs[j];
    memset(&s, 0, sizeof(s));
    s.cell_codes = own[p.cell];
    s.cell_labels = gd[p.cell].labels;
    s.codes = gcodes + r0 * 8;
    s.labels = glab + r0;
    if (p.f) {
      s.kind = SUBSET_FILTER;
      s.bits = p.f->ids ? nullptr : p.f->bits;
      s.ids = p.f->ids;
      s.nwords = (p.f->n + 31) / 32;
    } else {
      s.kind = SUBSET_LIVE;
      s.bits = p.dead;
      s.n_rows = gd[p.cell].n;
      s.nwords = (s.n_rows + 31) / 32;
      if (!p.dead) {  // every row, read where it is (the kernels only read a subset's codes and labels)
        s.codes = const_cast<uint8_t *>(s.cell_codes);
        s.labels = const_cast<uint64_t *>(s.cell_labels);
      }
    }
    s.block_offs = boffs + bl0;
    s.n = plan_rows(p);
    s.queries = dq + hq.size();
    s.nq = (int32_t)p.rows.size();
    s.k = p.k;
    s.cell = p.cell;
    if (s.bits || s.ids) r0 += s.n;
    if (s.bits) bl0 += (s.nwords + 255) / 256;
    hq.insert(hq.end(), p.rows.begin(), p.rows.end());
    cs->last_scanned_pairs += s.nq;
    cs->last_scanned_rows += (int64_t)s.nq * s.n;
  }
  ANNB_CUDA(cudaMemcpyAsync(djobs, jobs.data(), J * sizeof(SubsetScan), cudaMemcpyHostToDevice, st));
  ANNB_CUDA(cudaMemcpyAsync(dq, hq.data(), hq.size() * 4, cudaMemcpyHostToDevice, st));
  ANNB_CUDA(cudaMemcpyAsync(dtiles, tiles.data(), tiles.size() * sizeof(int4), cudaMemcpyHostToDevice, st));
  ss.djobs = djobs;
  ss.dtiles = dtiles;
  return ANNB_OK;  // (pageable sources: each copy has taken its data when it returns)
}

// the staged scans, after the fused walk (which writes the rows of the pairs it skips): results into the by-cell scratch
int launch_scans(annb_cellset *cs, const StagedScans &ss, const float *tables, const Staged &b, int limit) {
  for (size_t g = 0; g < ss.groups.size(); g++) {
    const size_t j0 = ss.groups[g].first, j1 = ss.groups[g].second;
    const std::vector<SubsetScan> part(ss.jobs.begin() + (ptrdiff_t)j0, ss.jobs.begin() + (ptrdiff_t)j1);
    const SubsetChunks &ch = ss.chunks[g];
    if (ch.rows) ANNB_CUDA(cudaMemsetAsync(ch.done, 0, (size_t)ss.tile_groups[g] * 4, cs->h0->stream));
    ANNB_TRY_RC(launch_subset_scan(cs->h0, cs->h0->stream, ss.djobs + j0, part, ss.dtiles + ss.tile0[g], ss.tile0[g + 1] - ss.tile0[g],
                                   ch, tables, cs->n_cells, limit, b.sl, b.sd, b.sfound, b.sstats));
  }
  return ANNB_OK;
}

// cell c is scanned: the scan's geometry and the cell's own codes are checked / made current here
int scan_cell(annb_cellset *cs, int c, std::vector<const uint8_t *> &own) {
  if (own[(size_t)c]) return ANNB_OK;
  annb_index *h = cs->cells[(size_t)c];
  if (!subset_scan_applicable(h))
    ANNB_FAIL(ANNB_ELIMIT, "cell %d: the exact subset scan needs M = 8 one-byte codes with 256 centroids", c);
  return sync_own_codes(h, &own[(size_t)c]);
}

// cell c's filter `f` is scanned rather than walked: its threshold is set (ANNB_CELLS_EXACT: +inf) and the filter
// admits at most that many (`need_rows`: and at least one)
int scan_decision(annb_cellset *cs, int c, const PreparedFilter *f, bool need_rows, bool exact, std::vector<const uint8_t *> &own,
                  bool *out) {
  const int64_t lim = exact ? INT64_MAX : (cs->below.empty() ? -1 : cs->below[(size_t)c]);
  *out = lim >= 0 && f->count <= lim && (!need_rows || f->count > 0);
  return *out ? scan_cell(cs, c, own) : ANNB_OK;
}

// The argument checks of a cell-set search: `bad` = the entry point's own check of B, limit, ef and its pointers,
// failing with `what`; `pair_limit` = B x n_cells must stay below 2^31 (the per-pair tables of the per-query form)
int check_search(annb_cellset *cs, bool bad, const char *what, bool pair_limit, int64_t B, const int32_t *order, int in_space,
                 int n_probe, int limit, int ef) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  const int C = cs->n_cells;
  if (bad) ANNB_FAIL(ANNB_EINVAL, "%s", what);
  if (n_probe < 1 || n_probe > C) ANNB_FAIL(ANNB_EINVAL, "n_probe=%d outside 1..n_cells=%d", n_probe, C);
  if (!order && !cs->d_centroids) ANNB_FAIL(ANNB_ESTATE, "no centroids: pass the probe order");
  const int ef_max = std::max(ef, limit);
  if (ef_max > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "max(ef, limit)=%d exceeds ANNB_MAX_EF=%d", ef_max, ANNB_MAX_EF);
  if (pair_limit && (double)B * C >= 2147483647.0) ANNB_FAIL(ANNB_ELIMIT, "B x n_cells=%lld exceeds 2^31-1", (long long)B * C);
  if (order && in_space != ANNB_DEVICE) ANNB_TRY_RC(check_order(order, B, n_probe, C));
  return ANNB_OK;
}

// Every cell's device graph brought up to date, its streams drained and its descriptor read now (buffers move on
// resize, nothing is cached), then step(c, h) under the same lock: what the search resolves against that snapshot
template <class Step>
int sync_cells(annb_cellset *cs, std::vector<GraphDev> &gd, Step step) {
  ANNB_CUDA(cudaSetDevice(cs->h0->device));
  gd.resize((size_t)cs->n_cells);
  for (int c = 0; c < cs->n_cells; c++) {
    annb_index *h = cs->cells[(size_t)c];
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->g.inited) ANNB_FAIL(ANNB_ESTATE, "cell %d: index not initialised", c);
    ANNB_TRY_RC(sync_device_graph(h));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream2));
    gd[(size_t)c] = h->gd;
    ANNB_TRY_RC(step(c, h));
  }
  return ANNB_OK;
}

// the K1 tables of the whole batch from its normalised queries, built on first use: for the scans, the cells' own
// launches and the re-runs
int batch_tables(annb_cellset *cs, Staged &b, int64_t B) {
  if (b.tables) return ANNB_OK;
  annb_index *h0 = cs->h0;
  ANNB_TRY_RC(cs_buf(cs, C_TABLES, (size_t)B * h0->M * h0->Ks * sizeof(float), (void **)&b.tables));
  std::lock_guard<std::mutex> lk(h0->mu);
  return launch_adc_table(h0, b.dq, B, b.tables);
}

// ANNB_CELLS_EXACT: the plans scanned and nothing walked, one launch for all of them (per_cell: one per cell), timed
// as the walk
int run_exact(annb_cellset *cs, Staged &b, int64_t B, int normalize, int limit, const std::vector<ScanPlan> &plans,
              const std::vector<const uint8_t *> &own, const std::vector<GraphDev> &gd, bool per_cell) {
  cudaStream_t st = cs->h0->stream;
  for (int r = 0; r < normalize; r++) ANNB_TRY_RC(launch_l2_normalize(cs->h0, b.dq, B, cs->dim));
  StagedScans ss;
  ANNB_TRY_RC(stage_scans(cs, plans, own, gd, per_cell, ss));
  if (!plans.empty()) ANNB_TRY_RC(batch_tables(cs, b, B));
  cudaEventRecord(cs->ev[2], st);
  if (!plans.empty()) ANNB_TRY_RC(launch_scans(cs, ss, b.tables, b, limit));
  cudaEventRecord(cs->ev[3], st);
  return ANNB_OK;
}

// One launch of cell c on its own handle's stream (after everything queued on the cell set's, which waits for it in
// turn), with k, mode and selectivity `sel`, its outputs scattered into the cell's rows of the by-cell scratch.  Query
// rows: every row (rows empty) or `rows`, which read the batch's tables through a query map (gather = false: the
// bitmap walk's re-run form) or from a gathered copy.  Filter: `filter` for every row, or qf[i] for row i (qf not empty).
int own_launch(annb_cellset *cs, Staged &b, int64_t B, int limit, int ef, int c, int mode, int k, float sel,
               const uint32_t *filter, const std::vector<uint32_t> &rows, const std::vector<const uint32_t *> &qf, bool gather) {
  annb_index *h = cs->cells[(size_t)c];
  cudaStream_t st = cs->h0->stream;
  const int TS = cs->h0->M * cs->h0->Ks;
  const int64_t n = rows.empty() ? B : (int64_t)rows.size();
  const int64_t out_rows = gather ? n : B;  // through a query map the walk writes row q of its outputs
  ANNB_TRY_RC(batch_tables(cs, b, B));
  uint64_t *tl;
  float *td, *gt = nullptr;
  int32_t *tf;
  int64_t *ts = nullptr;
  uint32_t *dmap = nullptr;
  const uint32_t **dqf = nullptr;
  ANNB_TRY_RC(cs_buf(cs, C_TMP_L, (size_t)out_rows * k * 8, (void **)&tl));
  ANNB_TRY_RC(cs_buf(cs, C_TMP_D, (size_t)out_rows * k * 4, (void **)&td));
  ANNB_TRY_RC(cs_buf(cs, C_TMP_F, (size_t)out_rows * 4, (void **)&tf));
  if (b.sstats) ANNB_TRY_RC(cs_buf(cs, C_TMP_S, (size_t)out_rows * 24, (void **)&ts));
  if (gather) ANNB_TRY_RC(cs_buf(cs, C_GTABLES, (size_t)n * TS * sizeof(float), (void **)&gt));
  if (!rows.empty()) {
    ANNB_TRY_RC(cs_buf(cs, C_QMAP, (size_t)n * 4, (void **)&dmap));
    ANNB_CUDA(cudaMemcpyAsync(dmap, rows.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  }
  if (!qf.empty()) {
    ANNB_TRY_RC(cs_buf(cs, C_QF, (size_t)n * sizeof(void *), (void **)&dqf));
    ANNB_CUDA(cudaMemcpyAsync(dqf, qf.data(), (size_t)n * sizeof(void *), cudaMemcpyHostToDevice, st));
  }
  SearchParams p;
  memset(&p, 0, sizeof(p));
  p.tables = gather ? gt : b.tables;
  p.qmap = gather ? nullptr : dmap;
  p.B = n;
  p.k = k;
  p.ef = std::max(ef, k);
  p.filter = filter;
  p.query_filter = dqf;
  p.selectivity = sel;
  p.out_labels = tl;
  p.out_dists = td;
  p.out_found = tf;
  p.out_stats = ts;
  std::lock_guard<std::mutex> lk(h->mu);
  ANNB_CUDA(cudaEventRecord(cs->ev[6], st));
  ANNB_CUDA(cudaStreamWaitEvent(h->stream, cs->ev[6], 0));
  if (gather) ANNB_TRY_RC(launch_rows_copy(h, b.tables, gt, dmap, n, TS, false));
  ANNB_TRY_RC(launch_search(h, p, mode));
  ANNB_TRY_RC(launch_cell_scatter(h->stream, tl, td, tf, ts, dmap, n, k, cs->n_cells, c, limit, b.sl, b.sd, b.sfound, b.sstats,
                                  gather));
  ANNB_CUDA(cudaEventRecord(cs->ev[7], h->stream));
  ANNB_CUDA(cudaStreamWaitEvent(st, cs->ev[7], 0));
  return ANNB_OK;
}

// The last pass of a filtered search over its walked pairs (walked[q * n_cells + c]): `found` read back; the pairs a
// walk flagged (found = -1) re-run on their cell's bitmap walk, one rerun(c, k, query rows) per (cell, k) with k =
// pair_k(q, c); `found` read back again if anything ran; then ANNB_EFEWRESULTS where a pair has fewer than its k
// results, as its cell's own search fails
template <class PairK, class Rerun>
int rerun_and_check(annb_cellset *cs, const Staged &b, int64_t B, const std::vector<char> &walked, PairK pair_k, Rerun rerun) {
  const int C = cs->n_cells;
  cudaStream_t st = cs->h0->stream;
  std::vector<int32_t> hfound((size_t)(B * C));
  ANNB_CUDA(cudaMemcpyAsync(hfound.data(), b.sfound, hfound.size() * 4, cudaMemcpyDeviceToHost, st));
  ANNB_CUDA(cudaStreamSynchronize(st));
  int64_t reruns = 0;
  for (int c = 0; c < C; c++) {
    std::map<int, std::vector<uint32_t>> over;
    for (int64_t q = 0; q < B; q++)
      if (walked[(size_t)(q * C + c)] && hfound[(size_t)(q * C + c)] < 0) over[pair_k(q, c)].push_back((uint32_t)q);
    for (auto &kv : over) {
      ANNB_TRY_RC(rerun(c, kv.first, kv.second));
      reruns += (int64_t)kv.second.size();
    }
  }
  cudaEventRecord(cs->ev[3], st);
  cs->last_rerun_pairs = reruns;
  if (reruns) {
    ANNB_CUDA(cudaMemcpyAsync(hfound.data(), b.sfound, hfound.size() * 4, cudaMemcpyDeviceToHost, st));
    ANNB_CUDA(cudaStreamSynchronize(st));
  }
  for (int64_t q = 0; q < B; q++)
    for (int c = 0; c < C; c++) {
      if (!walked[(size_t)(q * C + c)]) continue;
      const int k = pair_k(q, c);
      if (k > 0 && hfound[(size_t)(q * C + c)] < k)
        ANNB_FAIL(ANNB_EFEWRESULTS, "Cannot return the results in a contigious 2D array. Probably ef or M is too small");
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
  for (int i = 0; i < 8 && e == cudaSuccess; i++) e = cudaEventCreate(&cs->ev[i]);
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
  ANNB_TRY_RC(check_search(cs, B < 0 || limit <= 0 || ef <= 0 || !labels_out || !dists_out || !cells_out || (B > 0 && !queries),
                           "bad B / limit / ef / outputs", false, B, order, in_space, n_probe, limit, ef));
  const int C = cs->n_cells;
  annb_index *h0 = cs->h0;
  const bool exact = flags & ANNB_CELLS_EXACT;
  std::vector<GraphDev> gd;
  std::vector<int32_t> kc(C);
  std::vector<int64_t> live(C);
  std::vector<const uint32_t *> dead(C, nullptr);
  std::vector<const uint8_t *> own_codes(C, nullptr);
  bool fused = !(flags & ANNB_CELLS_GENERIC);
  ANNB_TRY_RC(sync_cells(cs, gd, [&](int c, annb_index *h) {
    live[c] = std::max<int64_t>(h->g.count.load() - h->g.num_deleted, 0);
    kc[c] = (int32_t)std::min<int64_t>(limit, live[c]);  // container.py:104-105, :119
    if (exact) {
      if (h->g.num_deleted > 0) dead[c] = gd[c].deleted;
      return kc[c] > 0 || !subset_scan_applicable(h) ? scan_cell(cs, c, own_codes) : ANNB_OK;
    }
    fused &= h->g.num_deleted == 0 && !h->opt_force_general && walk4_can_fuse(h) && h->M == 8;
    return ANNB_OK;
  }));
  cs->last_route = fused ? 0 : 1;
  cs->last_scanned_pairs = 0;
  cs->last_scanned_rows = 0;
  if (B == 0) return ANNB_OK;
  cudaStream_t st = h0->stream;
  Staged b;
  ANNB_TRY_RC(stage_batch(cs, queries, in_space, B, order, n_probe, limit, part_stats != nullptr, b));
  if (exact) {
    // every probed cell with k > 0 scanned over its live rows for the queries that probe it
    std::vector<int32_t> otmp;
    const int32_t *ho;
    ANNB_TRY_RC(host_order(cs, order, in_space, b.dorder, B, n_probe, otmp, &ho));
    std::vector<ScanPlan> plans(C);
    for (int c = 0; c < C; c++) {
      plans[c].cell = c;
      plans[c].k = kc[c];
      plans[c].live = live[c];
      plans[c].dead = dead[c];
    }
    for (int64_t q = 0; q < B; q++)
      for (int i = 0; i < n_probe; i++) plans[(size_t)ho[q * n_probe + i]].rows.push_back((uint32_t)q);
    std::vector<ScanPlan> kept;
    for (ScanPlan &p : plans)
      if (p.k > 0 && !p.rows.empty()) kept.push_back(std::move(p));
    ANNB_TRY_RC(run_exact(cs, b, B, normalize, limit, kept, own_codes, gd, !fused));
    return merge_and_finish(cs, b.sd, b.sl, b.sfound, b.sstats, b.dorder, !order, B, n_probe, limit, labels_out, dists_out, cells_out,
                            out_space, part_labels, part_dists, part_stats);
  }
  float *dq = b.dq;
  int32_t *dorder = b.dorder, *sfound = b.sfound;
  uint64_t *sl = b.sl;
  float *sd = b.sd;
  int64_t *sstats = b.sstats;
  if (fused) {
    for (int r = 0; r < normalize; r++) ANNB_TRY_RC(launch_l2_normalize(h0, dq, B, cs->dim));
    int32_t *dk;
    ANNB_TRY_RC(cs_buf(cs, C_K, (size_t)C * 4, (void **)&dk));
    ANNB_CUDA(cudaMemcpyAsync(cs->d_graphs, gd.data(), sizeof(GraphDev) * C, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dk, kc.data(), (size_t)C * 4, cudaMemcpyHostToDevice, st));
    SearchParams p;
    cells_params(cs, b, B, n_probe, limit, ef, dk, p);
    std::lock_guard<std::mutex> lk(h0->mu);
    cudaEventRecord(cs->ev[2], st);
    const int rc = launch_walk4_cells(h0, p);
    if (rc == 1) ANNB_FAIL(ANNB_ESTATE, "the multi-cell walk does not apply to these cells");
    if (rc) return rc;
    cudaEventRecord(cs->ev[3], st);
  } else {
    // generic route: one annb_search per probed cell over the whole batch (deletion-aware, any geometry), its
    // outputs copied into the cell's slot of the scratch
    ANNB_TRY_RC(per_cell_route(cs, order, in_space, dorder, B, n_probe, limit, kc, sl, sd, sfound, sstats,
                               [&](int c, int k, uint64_t *hl, float *hd, int64_t *hs) {
                                 const int rc = annb_search(cs->cells[c], queries, nullptr, in_space, B, normalize, k, ef, nullptr,
                                                            ANNB_HOST, 0, hl, hd, ANNB_HOST, hs);
                                 return rc == ANNB_EFEWRESULTS ? ANNB_OK : rc;  // a short row is padded with UINT64_MAX: the merge stops there
                               }));
  }
  return merge_and_finish(cs, sd, sl, sfound, sstats, dorder, !order, B, n_probe, limit, labels_out, dists_out, cells_out, out_space,
                          part_labels, part_dists, part_stats);
}

// The filtered search over a cell set: cell c admits the rows of its handle's prepared filter filter_ids[c] (0 = none).
// Per cell: k_c = min(limit, admitted rows, live rows), ef_c = max(ef, k_c), what annb_search_prepared does for the cell
// alone with k_c.  Fused route (every cell M = 8, 256 u8 codes, hnsw_walk4f geometry for max(ef, limit)): one launch of
// hnsw_walk4f's multi-cell form over every cell whose selectivity hnsw_walk4f covers for its ef_c, N sized for the most
// selective of them; each other cell gets the filtered launch annb_search_prepared would run for it (hnsw_walk_flagged or
// the bitmap walk over K1 tables, the whole batch) on its own handle; (query, cell) pairs any walk flagged are re-run on
// the bitmap walk of their cell.  Everything runs on the device into the by-cell scratch, then the merge.
int annb_cellset_search_prepared(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int normalize,
                                 const int32_t *order, int n_probe, int limit, int ef, int flags, const int *filter_ids,
                                 uint64_t *labels_out, float *dists_out, int32_t *cells_out, int out_space,
                                 uint64_t *part_labels, float *part_dists, int64_t *part_stats) {
  ANNB_TRY_RC(check_search(cs,
                           B < 0 || limit <= 0 || ef <= 0 || !labels_out || !dists_out || !cells_out || (B > 0 && !queries) ||
                               !filter_ids,
                           "bad B / limit / ef / outputs / filter ids", false, B, order, in_space, n_probe, limit, ef));
  const int C = cs->n_cells;
  const int ef_max = std::max(ef, limit);
  annb_index *h0 = cs->h0;
  std::vector<GraphDev> gd;
  std::vector<int32_t> kc(C, 0);
  std::vector<const uint32_t *> bits(C, nullptr);
  std::vector<float> sel(C, 0.f);
  std::vector<const PreparedFilter *> pfs(C, nullptr);
  std::vector<char> scan(C, 0);  // 1 = the cell's subset is scanned exactly (annb_cellset_set_bruteforce)
  std::vector<const uint8_t *> own_codes(C, nullptr);
  const bool exact = flags & ANNB_CELLS_EXACT;
  bool fused = !(flags & ANNB_CELLS_GENERIC);
  ANNB_TRY_RC(sync_cells(cs, gd, [&](int c, annb_index *h) {
    if (exact && !subset_scan_applicable(h)) return scan_cell(cs, c, own_codes);  // (fails: the scan's geometry)
    if (filter_ids[c] != 0) {
      PreparedFilter *f;
      const int rc = find_prepared_filter(h, filter_ids[c], &f);
      if (rc) {
        const std::string msg = annb_last_error();
        ANNB_FAIL(rc, "cell %d: %s", c, msg.c_str());
      }
      const int64_t live = h->g.count.load() - h->g.num_deleted;
      kc[c] = (int32_t)std::min<int64_t>({(int64_t)limit, f->count, std::max<int64_t>(live, 0)});
      bits[c] = f->bits;
      // the selectivity annb_search_prepared sizes the cell's lists by (SearchParams::selectivity is fp32)
      sel[c] = (float)search_selectivity(h, true, f->count);
      pfs[c] = f;
      bool sc;
      ANNB_TRY_RC(scan_decision(cs, c, f, true, exact, own_codes, &sc));
      scan[c] = sc;
    }
    int ep, en;
    if (!exact) fused &= walk4_can_fuse(h) && h->M == 8 && h->opt_force_general != 2 && walk4f_geometry(h, ef_max, 1.0, &ep, &en);
    return ANNB_OK;
  }));
  // fused route: the cells hnsw_walk4f serves, and N's size (the largest any of them needs alone)
  std::vector<char> own(C, 0);  // 1 = the cell's own filtered launch
  int ep = ef_max <= 64 ? 2 : 4, en = 0, n_own = 0;
  if (fused) {
    for (int c = 0; c < C; c++) {
      if (kc[c] == 0 || scan[c]) continue;
      int ep_c, en_c;
      if (walk4f_geometry(cs->cells[c], std::max(ef, kc[c]), (double)sel[c], &ep_c, &en_c)) {
        en = std::max(en, en_c);
      } else {
        own[c] = 1;
        n_own++;
      }
    }
    if (en > 0) en = walk4f_round_en(ep, en);
  }
  cs->last_route = fused ? 0 : 1;
  cs->last_rerun_pairs = 0;
  cs->last_handle_cells = 0;
  cs->last_scanned_pairs = 0;
  cs->last_scanned_rows = 0;
  if (B == 0) return ANNB_OK;
  cudaStream_t st = h0->stream;
  Staged b;
  ANNB_TRY_RC(stage_batch(cs, queries, in_space, B, order, n_probe, limit, part_stats != nullptr, b));
  // the scanned cells: every query that probes one scans its subset with k_c (annb_scan_subset over the whole batch in
  // the per-cell route; the merge reads only the probing queries' rows)
  std::vector<ScanPlan> plans;
  bool any_scan = false;
  for (int c = 0; c < C; c++) any_scan |= scan[c] && kc[c] > 0;
  if (any_scan) {
    std::vector<int32_t> otmp;
    const int32_t *ho;
    ANNB_TRY_RC(host_order(cs, order, in_space, b.dorder, B, n_probe, otmp, &ho));
    std::vector<int> at(C, -1);
    for (int c = 0; c < C; c++)
      if (scan[c] && kc[c] > 0) {
        at[c] = (int)plans.size();
        plans.emplace_back();
        plans.back().cell = c;
        plans.back().k = kc[c];
        plans.back().f = pfs[c];
      }
    for (int64_t q = 0; q < B; q++)
      for (int i = 0; i < n_probe; i++) {
        const int c = ho[q * n_probe + i];
        if (at[c] >= 0) plans[(size_t)at[c]].rows.push_back((uint32_t)q);
      }
    ANNB_TRY_RC(check_plans(plans));
  }
  if (exact) {
    ANNB_TRY_RC(run_exact(cs, b, B, normalize, limit, plans, own_codes, gd, !fused));
  } else if (!fused) {
    // one annb_search_prepared per probed cell that is not scanned; a walk with fewer than k_c results fails the call as
    // it fails the cell
    std::vector<int32_t> kpc(kc);
    for (int c = 0; c < C; c++)
      if (scan[c]) kpc[c] = 0;
    ANNB_TRY_RC(per_cell_route(cs, order, in_space, b.dorder, B, n_probe, limit, kpc, b.sl, b.sd, b.sfound, b.sstats,
                               [&](int c, int k, uint64_t *hl, float *hd, int64_t *hs) {
                                 return search_prepared_stats(cs->cells[c], queries, in_space, B, normalize, k, ef, filter_ids[c],
                                                              hl, hd, ANNB_HOST, hs);
                               }));
    if (!plans.empty()) {  // one scan launch per scanned cell, on the device
      for (int r = 0; r < normalize; r++) ANNB_TRY_RC(launch_l2_normalize(h0, b.dq, B, cs->dim));
      StagedScans ss;
      ANNB_TRY_RC(stage_scans(cs, plans, own_codes, gd, true, ss));
      ANNB_TRY_RC(batch_tables(cs, b, B));
      ANNB_TRY_RC(launch_scans(cs, ss, b.tables, b, limit));
      cudaEventRecord(cs->ev[3], st);
    }
  } else {
    for (int r = 0; r < normalize; r++) ANNB_TRY_RC(launch_l2_normalize(h0, b.dq, B, cs->dim));
    std::vector<int32_t> kwalk(kc);
    for (int c = 0; c < C; c++)
      if (own[c] || scan[c]) kwalk[c] = 0;
    int32_t *dk;
    const uint32_t **dbits;
    ANNB_TRY_RC(cs_buf(cs, C_K, (size_t)C * 4, (void **)&dk));
    ANNB_TRY_RC(cs_buf(cs, C_BITS, (size_t)C * sizeof(void *), (void **)&dbits));
    ANNB_CUDA(cudaMemcpyAsync(cs->d_graphs, gd.data(), sizeof(GraphDev) * C, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dk, kwalk.data(), (size_t)C * 4, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dbits, bits.data(), (size_t)C * sizeof(void *), cudaMemcpyHostToDevice, st));
    std::vector<int32_t> otmp;
    const int32_t *ho;
    ANNB_TRY_RC(host_order(cs, order, in_space, b.dorder, B, n_probe, otmp, &ho));
    StagedScans ss;
    ANNB_TRY_RC(stage_scans(cs, plans, own_codes, gd, false, ss));
    if (!plans.empty()) ANNB_TRY_RC(batch_tables(cs, b, B));
    cudaEventRecord(cs->ev[2], st);
    if (en > 0) {
      SearchParams p;
      cells_params(cs, b, B, n_probe, limit, ef, dk, p);
      p.cell_filter = dbits;
      std::lock_guard<std::mutex> lk(h0->mu);
      const int rc = launch_walk4f_cells(h0, p, ep, en);
      if (rc == 1) ANNB_FAIL(ANNB_ESTATE, "the filtered multi-cell walk does not apply to these cells");
      if (rc) return rc;
    }
    // the scans, one launch for every scanned cell
    if (!plans.empty()) ANNB_TRY_RC(launch_scans(cs, ss, b.tables, b, limit));
    // the cells on their own filtered launch: the whole batch, as the per-cell search walks it
    const std::vector<uint32_t> every_row;
    const std::vector<const uint32_t *> no_qf;
    std::vector<char> probed(C, 0);
    for (int64_t i = 0; i < B * n_probe; i++) probed[ho[i]] = 1;
    for (int c = 0; c < C; c++) {
      if (!own[c] || !probed[c]) continue;
      ANNB_TRY_RC(own_launch(cs, b, B, limit, ef, c, 1, kc[c], sel[c], bits[c], every_row, no_qf, false));
      cs->last_handle_cells++;
    }
    // the walked pairs (a cell on its own launch walked every query, as the per-cell search does: all its rows count);
    // flagged ones re-run cell by cell on the batch's tables through a query map
    std::vector<char> walked((size_t)B * C, 0);
    for (int64_t q = 0; q < B; q++) {
      for (int i = 0; i < n_probe; i++) walked[q * C + ho[q * n_probe + i]] = !scan[ho[q * n_probe + i]];
      for (int c = 0; c < C; c++)
        if (own[c] && probed[c]) walked[q * C + c] = 1;
    }
    ANNB_TRY_RC(rerun_and_check(cs, b, B, walked, [&](int64_t, int c) { return kc[c]; },
                                [&](int c, int k, const std::vector<uint32_t> &rows) {
                                  return own_launch(cs, b, B, limit, ef, c, 2, k, sel[c], bits[c], rows, no_qf, false);
                                }));
  }
  return merge_and_finish(cs, b.sd, b.sl, b.sfound, b.sstats, b.dorder, !order, B, n_probe, limit, labels_out, dists_out, cells_out,
                          out_space, part_labels, part_dists, part_stats);
}

// The search over a cell set with a filter per query: query q admits in cell c the rows of cell c's prepared filter
// query_filter[q * n_cells + c] (0 = no filter there: the live rows).  Each (query, cell) pair is what
// annb_search_multi does for that query on that cell alone, with k = min(limit, admitted rows, live rows) (no filter:
// min(limit, live rows)) and ef = max(ef, k).  Identical rows of the id table share a slot, so the walk's per-pair
// tables are (slots, n_cells).  Fused route (every cell M = 8, 256 u8 codes, hnsw_walk4f geometry for max(ef, limit)):
// one launch of hnsw_walk4f's per-query multi-cell form over every probed pair whose selectivity hnsw_walk4f covers at
// its ef, N sized for the most selective of them; the other pairs get their cell's own launch over their rows (the
// kernel annb_search_multi picks for them, over K1 tables, one launch per distinct k and kind of filter); pairs any walk
// flagged are re-run on their cell's bitmap walk with their own bitmap.  Other geometries, ef > 128 and
// ANNB_CELLS_GENERIC send every pair to its cell's own launch.  Everything runs on the device, then the merge.
int annb_cellset_search_multi(annb_cellset_t *cs, const float *queries, int in_space, int64_t B, int normalize,
                              const int32_t *order, int n_probe, int limit, int ef, int flags, const int *query_filter,
                              uint64_t *labels_out, float *dists_out, int32_t *cells_out, int out_space,
                              uint64_t *part_labels, float *part_dists, int64_t *part_stats) {
  ANNB_TRY_RC(check_search(cs,
                           B < 0 || limit <= 0 || ef <= 0 || !labels_out || !dists_out || !cells_out || (B > 0 && !queries) ||
                               !query_filter,
                           "bad B / limit / ef / outputs / filter ids", true, B, order, in_space, n_probe, limit, ef));
  const int C = cs->n_cells;
  const int ef_max = std::max(ef, limit);
  annb_index *h0 = cs->h0;
  // slots: the distinct rows of the id table, each represented by its first query
  std::vector<int32_t> slot((size_t)B);
  std::vector<int64_t> srep;
  {
    std::unordered_map<std::string, int32_t> seen;
    for (int64_t q = 0; q < B; q++) {
      auto it = seen.emplace(std::string((const char *)(query_filter + q * C), (size_t)C * sizeof(int)), (int32_t)srep.size());
      if (it.second) srep.push_back(q);
      slot[(size_t)q] = it.first->second;
    }
  }
  const int64_t S = (int64_t)srep.size();
  auto row_id = [&](int64_t s, int c) { return query_filter[srep[(size_t)s] * C + c]; };
  // every cell's device graph up to date, its filters resolved; per (slot, cell): k, bitmap, selectivity
  std::vector<GraphDev> gd;
  std::vector<int64_t> ndel(C);
  std::vector<int32_t> sk((size_t)(S * C), 0);
  std::vector<const uint32_t *> sbits((size_t)(S * C), nullptr);  // nullptr = no filter in this cell
  std::vector<float> ssel((size_t)(S * C), 1.f);
  std::vector<const PreparedFilter *> spf((size_t)(S * C), nullptr);
  std::vector<char> sscan((size_t)(S * C), 0);  // 1 = the pair's subset is scanned exactly (annb_cellset_set_bruteforce)
  std::vector<const uint8_t *> own_codes(C, nullptr);
  std::vector<int64_t> nlive(C);
  const bool exact = flags & ANNB_CELLS_EXACT;
  bool fused = !(flags & ANNB_CELLS_GENERIC);
  ANNB_TRY_RC(sync_cells(cs, gd, [&](int c, annb_index *h) {
    if (exact && !subset_scan_applicable(h)) return scan_cell(cs, c, own_codes);  // (fails: the scan's geometry)
    ndel[c] = h->g.num_deleted;
    const int64_t live = std::max<int64_t>(h->g.count.load() - h->g.num_deleted, 0);
    nlive[c] = live;
    std::unordered_map<int, const PreparedFilter *> pf;
    for (int64_t s = 0; s < S; s++) {
      const int id = row_id(s, c);
      const size_t i = (size_t)(s * C + c);
      if (id == 0) {  // annb_search_multi's unfiltered rows: the live rows (k = min(limit, live), container.py:119)
        sk[i] = (int32_t)std::min<int64_t>(limit, live);
        ssel[i] = (float)search_selectivity(h, false, 0);
        if (exact && sk[i] > 0) {  // ANNB_CELLS_EXACT: scanned over the cell's live rows
          sscan[i] = 1;
          ANNB_TRY_RC(scan_cell(cs, c, own_codes));
        }
        continue;
      }
      auto it = pf.find(id);
      if (it == pf.end()) {
        PreparedFilter *f;
        const int rc = find_prepared_filter(h, id, &f);
        if (rc) {
          const std::string msg = annb_last_error();
          ANNB_FAIL(rc, "cell %d: %s", c, msg.c_str());
        }
        if ((int)pf.size() >= ANNB_FILTER_MAX_PER_CALL)
          ANNB_FAIL(ANNB_ELIMIT, "cell %d: more than %d distinct filters in one call", c, ANNB_FILTER_MAX_PER_CALL);
        it = pf.emplace(id, f).first;
      }
      const PreparedFilter *f = it->second;
      sk[i] = (int32_t)std::min<int64_t>({(int64_t)limit, f->count, live});
      sbits[i] = f->bits;
      ssel[i] = (float)search_selectivity(h, true, f->count);
      spf[i] = f;
      bool sc;
      ANNB_TRY_RC(scan_decision(cs, c, f, false, exact, own_codes, &sc));
      sscan[i] = sc;
    }
    int ep, en;
    if (!exact) fused &= walk4_can_fuse(h) && h->M == 8 && h->opt_force_general != 2 && walk4f_geometry(h, ef_max, 1.0, &ep, &en);
    return ANNB_OK;
  }));
  cs->last_route = fused ? 0 : 1;
  cs->last_rerun_pairs = 0;
  cs->last_handle_cells = 0;
  cs->last_scanned_pairs = 0;
  cs->last_scanned_rows = 0;
  if (B == 0) return ANNB_OK;
  cudaStream_t st = h0->stream;
  Staged b;
  ANNB_TRY_RC(stage_batch(cs, queries, in_space, B, order, n_probe, limit, part_stats != nullptr, b));
  if (!exact)
    for (int r = 0; r < normalize; r++) ANNB_TRY_RC(launch_l2_normalize(h0, b.dq, B, cs->dim));
  std::vector<int32_t> otmp;
  const int32_t *ho;
  ANNB_TRY_RC(host_order(cs, order, in_space, b.dorder, B, n_probe, otmp, &ho));
  // the pairs walked: probed, with k > 0, not scanned (and which slots probe which cells); the scanned ones: one plan per
  // (cell, filter), its queries in batch order
  std::vector<char> walked((size_t)(B * C), 0), sprobed((size_t)(S * C), 0);
  std::map<std::pair<int, int>, ScanPlan> by_filter;
  for (int64_t q = 0; q < B; q++)
    for (int i = 0; i < n_probe; i++) {
      const int c = ho[q * n_probe + i];
      const size_t sc = (size_t)slot[(size_t)q] * C + c;
      sprobed[sc] = 1;
      walked[(size_t)(q * C + c)] = sk[sc] > 0 && !sscan[sc];
      if (sk[sc] > 0 && sscan[sc]) {
        ScanPlan &pl = by_filter[{c, row_id(slot[(size_t)q], c)}];
        pl.cell = c;
        pl.k = sk[sc];
        pl.f = spf[sc];  // (nullptr: no filter, the live rows)
        pl.live = nlive[c];
        pl.dead = ndel[c] > 0 ? gd[c].deleted : nullptr;
        pl.rows.push_back((uint32_t)q);
      }
    }
  std::vector<ScanPlan> plans;
  for (auto &kv : by_filter) plans.push_back(std::move(kv.second));
  ANNB_TRY_RC(check_plans(plans));
  if (exact) {
    ANNB_TRY_RC(run_exact(cs, b, B, normalize, limit, plans, own_codes, gd, !fused));
    return merge_and_finish(cs, b.sd, b.sl, b.sfound, b.sstats, b.dorder, !order, B, n_probe, limit, labels_out, dists_out, cells_out,
                            out_space, part_labels, part_dists, part_stats);
  }
  // fused route: the pairs hnsw_walk4f serves, and N's size (the largest any of them needs alone)
  std::vector<char> own((size_t)(S * C), 0);  // 1 = the pair goes to its cell's own launch
  int ep = ef_max <= 64 ? 2 : 4, en = 0;
  for (int64_t s = 0; s < S; s++)
    for (int c = 0; c < C; c++) {
      const size_t i = (size_t)(s * C + c);
      if (!sprobed[i] || sk[i] == 0 || sscan[i]) continue;
      int ep_c, en_c;
      if (fused && walk4f_geometry(cs->cells[c], std::max(ef, sk[i]), (double)ssel[i], &ep_c, &en_c)) en = std::max(en, en_c);
      else own[i] = 1;
    }
  if (en > 0) en = walk4f_round_en(ep, en);
  StagedScans ss;
  ANNB_TRY_RC(stage_scans(cs, plans, own_codes, gd, !fused, ss));
  if (!plans.empty()) ANNB_TRY_RC(batch_tables(cs, b, B));
  cudaEventRecord(cs->ev[2], st);
  if (en > 0) {
    // the walk's tables: k per (slot, cell) (0 = skip, own-launch pairs included) and the admission word: the filter's
    // bitmap, or (no filter) the cell's deletions read as "not deleted", with the size guard when there are any
    std::vector<int32_t> kwalk(sk);
    std::vector<uintptr_t> word((size_t)(S * C));
    for (size_t i = 0; i < word.size(); i++) {
      const int c = (int)(i % C);
      if (own[i] || sscan[i]) kwalk[i] = 0;
      const uint32_t *bits = sbits[i] ? sbits[i] : gd[c].deleted;  // (sync_device_graph always uploads the deletions)
      if (kwalk[i] > 0 && (!bits || (reinterpret_cast<uintptr_t>(bits) & 3u)))
        ANNB_FAIL(ANNB_ESTATE, "internal: cell %d has no 4-byte aligned admission bitmap", c);
      word[i] = reinterpret_cast<uintptr_t>(bits) | (sbits[i] ? 0u : 1u | (ndel[c] > 0 ? 2u : 0u));
    }
    int32_t *dslot, *dk;
    uintptr_t *dword;
    ANNB_TRY_RC(cs_buf(cs, C_SLOT, (size_t)B * 4, (void **)&dslot));
    ANNB_TRY_RC(cs_buf(cs, C_SLOT_K, kwalk.size() * 4, (void **)&dk));
    ANNB_TRY_RC(cs_buf(cs, C_SLOT_BITS, word.size() * sizeof(uintptr_t), (void **)&dword));
    ANNB_CUDA(cudaMemcpyAsync(cs->d_graphs, gd.data(), sizeof(GraphDev) * C, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dslot, slot.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dk, kwalk.data(), kwalk.size() * 4, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dword, word.data(), word.size() * sizeof(uintptr_t), cudaMemcpyHostToDevice, st));
    SearchParams p;
    cells_params(cs, b, B, n_probe, limit, ef, dk, p);
    p.cell_filter = reinterpret_cast<const uint32_t *const *>(dword);
    p.query_slot = dslot;
    std::lock_guard<std::mutex> lk(h0->mu);
    const int rc = launch_walk4f_cells(h0, p, ep, en);
    if (rc == 1) ANNB_FAIL(ANNB_ESTATE, "the per-query filtered multi-cell walk does not apply to these cells");
    if (rc) return rc;
  }
  // the scans, after the walk: one launch for all of them (ANNB_CELLS_GENERIC / other geometries: one per cell)
  if (!plans.empty()) ANNB_TRY_RC(launch_scans(cs, ss, b.tables, b, limit));
  // own launches, cell by cell, over their rows with the rows' tables gathered: one per (k, kind) -- kind 0 = no filter (annb_search_multi's plain or deletion-aware
  // group), 1 = filters hnsw_walk4f takes at that ef, 2 = the others -- as annb_search_multi groups the same rows
  for (int c = 0; c < C; c++) {
    annb_index *h = cs->cells[c];
    struct Group {
      std::vector<uint32_t> rows;
      std::vector<const uint32_t *> qf;
      double s = 1.0;
    };
    std::map<std::pair<int, int>, Group> groups;
    for (int64_t q = 0; q < B; q++) {
      const size_t i = (size_t)slot[(size_t)q] * C + c;
      if (!walked[(size_t)(q * C + c)] || !own[i]) continue;
      const int k = sk[i];
      bool walk4f = false;
      if (sbits[i]) search_route(h, std::max(ef, k), true, ssel[i], nullptr, &walk4f);
      const int kind = !sbits[i] ? 0 : (walk4f ? 1 : 2);
      Group &g = groups[{k, kind}];
      g.rows.push_back((uint32_t)q);
      if (kind) g.qf.push_back(sbits[i]);
      g.s = std::min(g.s, (double)ssel[i]);
    }
    for (auto &kv : groups) {
      const int k = kv.first.first, kind = kv.first.second;
      const int mode = search_route(h, std::max(ef, k), kind != 0, kv.second.s, nullptr, nullptr);
      ANNB_TRY_RC(own_launch(cs, b, B, limit, ef, c, mode, k, (float)kv.second.s, nullptr, kv.second.rows, kv.second.qf, true));
    }
    if (!groups.empty()) cs->last_handle_cells++;
  }
  // pairs a walk flagged: re-run on the bitmap walk of their cell with their own bitmap, one launch per (cell, k)
  auto pair_k = [&](int64_t q, int c) { return sk[(size_t)slot[(size_t)q] * C + c]; };
  ANNB_TRY_RC(rerun_and_check(cs, b, B, walked, pair_k, [&](int c, int k, const std::vector<uint32_t> &rows) {
    std::vector<const uint32_t *> qf(rows.size());
    for (size_t j = 0; j < rows.size(); j++) qf[j] = sbits[(size_t)slot[rows[j]] * C + c];
    return own_launch(cs, b, B, limit, ef, c, 2, k, 1.f, nullptr, rows, qf, true);
  }));
  return merge_and_finish(cs, b.sd, b.sl, b.sfound, b.sstats, b.dorder, !order, B, n_probe, limit, labels_out, dists_out, cells_out,
                          out_space, part_labels, part_dists, part_stats);
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

int annb_cellset_set_bruteforce(annb_cellset_t *cs, const int64_t *below) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (below)
    for (int c = 0; c < cs->n_cells; c++)
      if (below[c] < -1) ANNB_FAIL(ANNB_EINVAL, "cell %d: threshold %lld below -1", c, (long long)below[c]);
  cs->below.assign((size_t)cs->n_cells, -1);
  if (below) cs->below.assign(below, below + cs->n_cells);
  return ANNB_OK;
}

int annb_cellset_last_scanned(annb_cellset_t *cs, int64_t *pairs, int64_t *rows) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (pairs) *pairs = cs->last_scanned_pairs;
  if (rows) *rows = cs->last_scanned_rows;
  return ANNB_OK;
}

int annb_cellset_last_filtered(annb_cellset_t *cs, int64_t *rerun_pairs, int *handle_cells) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (rerun_pairs) *rerun_pairs = cs->last_rerun_pairs;
  if (handle_cells) *handle_cells = cs->last_handle_cells;
  return ANNB_OK;
}

// Rows split by cell, each cell's share in input order.  A share that annb_add_items would build on the GPU (>= 16384
// fresh rows, no deletions, gpu_build_run's geometry) goes through gpu_build_cells together with the other such shares:
// phase 1 on a host thread per cell, phase 2 in rounds with one multi-cell walk and two link launches for all of them.
// Every other share is annb_add_items on its own handle.  Each cell's graph is what its own annb_add_items makes.
int annb_cellset_add_items(annb_cellset_t *cs, const float *vectors, const uint64_t *labels, const int32_t *cells, int64_t n,
                           int num_threads) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (n < 0 || (n > 0 && (!vectors || !labels || !cells))) ANNB_FAIL(ANNB_EINVAL, "null vectors/labels/cells");
  const int C = cs->n_cells;
  if (n > 0) ANNB_TRY_RC(check_finite_rows(vectors, n, cs->dim));
  std::vector<std::vector<int64_t>> rows((size_t)C);
  for (int64_t i = 0; i < n; i++) {
    const int32_t c = cells[i];
    if (c < 0 || c >= C) ANNB_FAIL(ANNB_EINVAL, "row %lld: %d is not a cell of the set (n_cells=%d)", (long long)i, c, C);
    rows[(size_t)c].push_back(i);
  }
  cs->build = CellBuildStats();
  cs->build_cells = 0;
  if (n == 0) return ANNB_OK;
  ANNB_CUDA(cudaSetDevice(cs->device));
  // every share is checked before anything is inserted
  std::vector<std::vector<uint64_t>> lab((size_t)C);
  std::vector<char> one_pass((size_t)C, 0);
  for (int c = 0; c < C; c++) {
    if (rows[c].empty()) continue;
    lab[c].resize(rows[c].size());
    for (size_t t = 0; t < rows[c].size(); t++) lab[c][t] = labels[rows[c][t]];
    annb_index *h = cs->cells[c];
    bool gpu;
    int rc;
    {
      std::lock_guard<std::mutex> lk(h->mu);
      rc = add_items_check(h, lab[c].data(), (int64_t)lab[c].size(), num_threads, &gpu);
    }
    if (rc) {
      const std::string msg = annb_last_error();
      ANNB_FAIL(rc, "cell %d: %s", c, msg.c_str());
    }
    // the multi-cell walk has the M = 8 geometry; one walk launch has one table form
    one_pass[c] = gpu && h->M == 8 && h->opt_ip_raw == cs->h0->opt_ip_raw;
  }
  std::vector<float> v;
  for (int c = 0; c < C; c++) {
    if (rows[c].empty() || one_pass[c]) continue;
    v.resize(rows[c].size() * (size_t)cs->dim);
    for (size_t t = 0; t < rows[c].size(); t++)
      memcpy(v.data() + t * cs->dim, vectors + (size_t)rows[c][t] * cs->dim, (size_t)cs->dim * 4);
    const int rc = annb_add_items(cs->cells[c], v.data(), nullptr, lab[c].data(), (int64_t)lab[c].size(), num_threads);
    if (rc) {
      const std::string msg = annb_last_error();
      ANNB_FAIL(rc, "cell %d: %s", c, msg.c_str());
    }
  }
  std::vector<CellBuildJob> jobs;
  for (int c = 0; c < C; c++) {
    if (!one_pass[c]) continue;
    jobs.emplace_back();
    CellBuildJob &j = jobs.back();
    j.h = cs->cells[c];
    j.cell = c;
    j.vectors = vectors;
    j.rows = std::move(rows[c]);
    j.labels = std::move(lab[c]);
  }
  if (jobs.empty()) return ANNB_OK;
  // cell 0's stream and scratch run phase 2: its lock is taken too (cells in ascending order)
  std::vector<std::unique_lock<std::mutex>> locks;
  if (!one_pass[0]) locks.emplace_back(cs->h0->mu);
  for (CellBuildJob &j : jobs) {
    locks.emplace_back(j.h->mu);
    const int rc = add_items_enter(j.h);
    if (rc) {
      const std::string msg = annb_last_error();
      ANNB_FAIL(rc, "cell %d: %s", j.cell, msg.c_str());
    }
  }
  ANNB_CUDA(cudaStreamSynchronize(cs->h0->stream));
  cs->build_cells = (int)jobs.size();
  return gpu_build_cells(cs->h0, jobs, num_threads, &cs->build);
}

int annb_cellset_last_build(annb_cellset_t *cs, double *phase1_ms, double *phase2_ms, int64_t *rounds, int *cells) {
  if (!cs) ANNB_FAIL(ANNB_EINVAL, "null cell set");
  if (phase1_ms) *phase1_ms = cs->build.phase1_ms;
  if (phase2_ms) *phase2_ms = cs->build.phase2_ms;
  if (rounds) *rounds = cs->build.rounds;
  if (cells) *cells = cs->build_cells;
  return ANNB_OK;
}

}  // extern "C"
