// gpu_build.cu -- batched HNSW insertion with the level-0 work on the GPU (SURVEY.md section 8f, rank 2, second half).
//
// Reference: addPoint (include/hnswlib/hnswalg.h:1108-1235) = greedy descent, then per level searchBaseLayer at
// ef_construction (:158-238), getNeighborsByHeuristic2 (:443-483) and mutuallyConnectNewElement (:502-619).  In PQ
// mode the reference's "distance between two stored nodes" is the distance from the point being inserted to the
// second node (PQLookup ignores its first argument, SURVEY.md section 0.2), which collapses the heuristic:
//   * the new node x links to the M_ nearest of its ef_construction candidates, farthest first;
//   * a selected neighbour r with room appends x; a full one keeps x and those of its neighbours that are NOT
//     closer to x than r itself is (in descending id order, at most maxM0 of them).
// hnsw_build.cpp restates that on the host, byte for byte.  Here the same rules run batch-wise on the device, with one
// difference of storage order: a rewritten list is stored here in descending id, while the reference's queue gives
// its entries (all of key d(x, r)) back in the pop order of an equal-key heap.  The set of links is the same; the
// order is kept so that a build, and every search over it, stays what earlier versions of this builder made.
//
//   phase 1 (host, existing code)  every node that owns upper-level lists (~1/M of the rows, levels drawn first with
//            the index's own generator) plus a few thousand level-0 rows are inserted by hnsw_insert_rows: the whole
//            upper hierarchy exists before phase 2 starts and is never touched again.
//   phase 2 (device) the remaining rows, all of level 0, in batches: PQ-encode (encode_kernel), ONE launch of the
//            search kernel itself (hnsw_walk4, table built in shared memory from the row's vector, ef = ef_construction,
//            k = M_, internal ids out) against the graph as it stood before the batch, then link_new_nodes_kernel
//            writes the new records and reverse_link_kernel applies the back-links, one warp per neighbour r taking
//            r's back-links in row order, evaluating "closer to x than r" directly from x's vector and the codebook
//            with the table's arithmetic.
//   finish   links and codes are exported, the host graph (reference byte layout: save_index, pickle state,
//            mark_deleted, further add_items all keep working) is assembled from them.
//
// Rows of one batch do not see each other as candidates (the multi-threaded reference has the same kind of race:
// concurrent insertions see a partially linked graph); batches grow with the graph (<= 1/16 of it by default, <= 65536 rows).
// The result is deterministic: phase 1 inserts on one host thread and phase 2 fixes the order of every write, so the
// same rows give the same graph on every run and machine, whatever num_threads is.
// The graph is NOT the one a sequential build makes, but every rule above is exact: tests/test_gpu_build_model.py
// compares the result byte for byte with a restatement of phase 2, which reproduces the sequential host build when
// its batches are one row and rewritten lists keep the reference's order (tests/test_build_model.py);
// tests/test_gpu_build.py checks the structural invariants, search parity over the result and recall against a
// host-built graph.
//
// gpu_build_cells runs the same build for the shares of a cell-set insertion together (annb_cellset_add_items):
// phase 1 on a host thread per cell, phase 2 in rounds where every cell inserts its next batch with one multi-cell walk
// launch and the multi-graph link kernels; each cell's graph is byte for byte what gpu_build_run makes of its share
// (tests/test_gpu_cells_build.py).
#include <math_constants.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <thread>

#include "annb_internal.h"

#define FULL_MASK 0xffffffffu

namespace {

#define EMPTY_LINK 0xffffffffu

// ADC distance of one stored code to the vector q, computed the way the table would: per subspace
// t = sum_j (cb - q)^2 (or cb*q) sequentially with separate roundings, then the sequential sum over m of
// t (L2) or bias - t (IP form): bit-identical to PQLookup over the K1 table.
__device__ __forceinline__ float adc_direct(const float *__restrict__ q, const float *__restrict__ cb, const uint8_t *code, int M,
                                            int ds, int is_ip, float bias) {
  float r = 0.f;
  for (int m = 0; m < M; m++) {
    const float *w = cb + ((size_t)m * 256 + code[m]) * ds;
    const float *x = q + m * ds;
    float acc = 0.f;
    if (!is_ip) {
      for (int j = 0; j < ds; j++) {
        const float t = __fsub_rn(__ldg(w + j), x[j]);
        acc = __fadd_rn(acc, __fmul_rn(t, t));
      }
    } else {
      for (int j = 0; j < ds; j++) acc = __fadd_rn(acc, __fmul_rn(__ldg(w + j), x[j]));
      acc = __fsub_rn(bias, acc);
    }
    r = __fadd_rn(r, acc);
  }
  return r;
}

struct BuildDev {
  uint8_t *rec0;           // level-0 walk records (mutable)
  uint64_t *labels;        // by internal id
  uint8_t *node_codes;     // (N, M) own code of every node
  int rec0_bytes, code_off0, maxM0, M;
};

// new node x = first + i: links = its `found` nearest candidates, FARTHEST first (connect(): sel is popped from a
// max-heap), neighbour codes co-located; label; own record otherwise empty
__global__ void link_new_nodes_kernel(BuildDev b, const uint64_t *__restrict__ sel, const int32_t *__restrict__ found, int k,
                                      const uint64_t *__restrict__ new_labels, uint32_t first, int B) {
  const int i = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= B) return;
  const uint32_t x = first + i;
  const int nf = min(found[i], k);
  uint8_t *rec = b.rec0 + (size_t)x * b.rec0_bytes;
  uint32_t link = EMPTY_LINK;
  if (lane < nf) link = (uint32_t)sel[(size_t)i * k + (nf - 1 - lane)];
  if (lane < b.maxM0) {
    reinterpret_cast<uint32_t *>(rec)[lane] = link;
    uint8_t *dst = rec + b.code_off0 + (size_t)lane * b.M;
    if (link != EMPTY_LINK) {
      const uint8_t *src = b.node_codes + (size_t)link * b.M;
      for (int t = 0; t < b.M; t++) dst[t] = src[t];
    } else {
      for (int t = 0; t < b.M; t++) dst[t] = 0;
    }
  }
  if (lane == 0) b.labels[x] = new_labels[i];
}

// back-links: one warp per neighbour r selected in this batch, applying r's back-links one after the other in row
// order (pairs p = i*k + j ascending, as a sequential insertion of the batch would): the graph a batch leaves does not
// depend on the order in which warps run.  rows / off / pairs: the host's counting sort of the batch's (r, p) pairs.
__global__ void reverse_link_kernel(BuildDev b, const uint32_t *__restrict__ rows, const uint32_t *__restrict__ off,
                                    const uint32_t *__restrict__ pairs, int R, const float *__restrict__ seld, int k,
                                    const float *__restrict__ q, int dim, const float *__restrict__ cb, int ds, int is_ip,
                                    float bias, uint32_t first) {
  const int w = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= R) return;
  const uint32_t r = rows[w];
  uint8_t *rec = b.rec0 + (size_t)r * b.rec0_bytes;
  volatile uint32_t *links = reinterpret_cast<volatile uint32_t *>(rec);
  volatile uint8_t *codes = rec + b.code_off0;
  const int M = b.M;
  for (uint32_t e = off[w]; e < off[w + 1]; e++) {
    const uint32_t p = pairs[e];
    const int i = (int)(p / (uint32_t)k);
    const uint32_t x = first + i;
    const float dr = seld[p];
    __syncwarp();  // the previous back-link's writes to r's record are visible to every lane
    uint32_t link = lane < b.maxM0 ? links[lane] : EMPTY_LINK;
    const bool valid = link != EMPTY_LINK;
    const int cnt = __popc(__ballot_sync(FULL_MASK, valid));
    const uint8_t *xcode = b.node_codes + (size_t)x * M;
    if (cnt < b.maxM0) {
      // room: append (hnswalg.h:575-578)
      if (lane == 0) links[cnt] = x;
      for (int t = lane; t < M; t += 32) codes[(size_t)cnt * M + t] = xcode[t];
    } else {
      // full: keep x and the neighbours that are not closer to x than r is; descending id, at most maxM0 (:579-616 in PQ mode)
      uint8_t mycode[128];
      for (int t = 0; t < M; t++) mycode[t] = valid ? codes[(size_t)lane * M + t] : 0;
      float d = CUDART_INF_F;
      if (valid) d = adc_direct(q + (size_t)i * dim, cb, mycode, M, ds, is_ip, bias);
      const bool keep = valid && !(d < dr);
      int rank = 0;
      for (int s = 0; s < 32; s++) {
        const uint32_t oid = __shfl_sync(FULL_MASK, link, s);
        const bool ok = __shfl_sync(FULL_MASK, (int)keep, s);
        rank += (ok && oid > link) ? 1 : 0;
      }
      const int nkeep = __popc(__ballot_sync(FULL_MASK, keep));
      const int total = min(1 + nkeep, b.maxM0);
      __syncwarp();  // every lane holds its old link and code in registers: the record may be rewritten
      if (keep && 1 + rank < b.maxM0) {
        links[1 + rank] = link;
        for (int t = 0; t < M; t++) codes[(size_t)(1 + rank) * M + t] = mycode[t];
      }
      if (lane == 0) {
        links[0] = x;
        for (int t = 0; t < M; t++) codes[t] = xcode[t];
      }
      if (lane >= total && lane < b.maxM0) links[lane] = EMPTY_LINK;
    }
  }
}

// ---- multi-graph forms (gpu_build_cells): one launch serves the batches of several graphs ------------------------
// Row i of a launch is inserted into graph row_cell[i] (descriptor bd[c], k = cell_k[c]) as node row_node[i].  The walk
// left its candidates in row i * n_cells + c of the by-cell scratch (`stride` entries per row), where they are read.

// link_new_nodes_kernel, per row of its own graph
__global__ void link_new_nodes_cells_kernel(const BuildDev *__restrict__ bd, const int32_t *__restrict__ cell_k,
                                            const int32_t *__restrict__ row_cell, const uint32_t *__restrict__ row_node,
                                            const uint64_t *__restrict__ sel, const int32_t *__restrict__ found, int n_cells,
                                            int stride, const uint64_t *__restrict__ new_labels, int B) {
  const int i = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= B) return;
  const int c = row_cell[i];
  const BuildDev b = bd[c];
  const int k = cell_k[c];
  const int64_t o = (int64_t)i * n_cells + c;
  const uint32_t x = row_node[i];
  const int nf = min(found[o], k);
  uint8_t *rec = b.rec0 + (size_t)x * b.rec0_bytes;
  uint32_t link = EMPTY_LINK;
  if (lane < nf) link = (uint32_t)sel[o * stride + (nf - 1 - lane)];
  if (lane < b.maxM0) {
    reinterpret_cast<uint32_t *>(rec)[lane] = link;
    uint8_t *dst = rec + b.code_off0 + (size_t)lane * b.M;
    if (link != EMPTY_LINK) {
      const uint8_t *src = b.node_codes + (size_t)link * b.M;
      for (int t = 0; t < b.M; t++) dst[t] = src[t];
    } else {
      for (int t = 0; t < b.M; t++) dst[t] = 0;
    }
  }
  if (lane == 0) b.labels[x] = new_labels[i];
}

// reverse_link_kernel, per neighbour r of graph rcell[w]; a pair p = i * stride + j is candidate j of launch row i
__global__ void reverse_link_cells_kernel(const BuildDev *__restrict__ bd, const int32_t *__restrict__ rcell,
                                          const uint32_t *__restrict__ rows, const uint32_t *__restrict__ off,
                                          const uint32_t *__restrict__ pairs, int R, const float *__restrict__ seld,
                                          const uint32_t *__restrict__ row_node, int n_cells, int stride,
                                          const float *__restrict__ q, int dim, const float *__restrict__ cb, int ds, int is_ip,
                                          float bias) {
  const int w = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= R) return;
  const int c = rcell[w];
  const BuildDev b = bd[c];
  const uint32_t r = rows[w];
  uint8_t *rec = b.rec0 + (size_t)r * b.rec0_bytes;
  volatile uint32_t *links = reinterpret_cast<volatile uint32_t *>(rec);
  volatile uint8_t *codes = rec + b.code_off0;
  const int M = b.M;
  for (uint32_t e = off[w]; e < off[w + 1]; e++) {
    const uint32_t p = pairs[e];
    const int i = (int)(p / (uint32_t)stride);
    const int j = (int)(p - (uint32_t)i * (uint32_t)stride);
    const uint32_t x = row_node[i];
    const float dr = seld[((int64_t)i * n_cells + c) * stride + j];
    __syncwarp();  // the previous back-link's writes to r's record are visible to every lane
    uint32_t link = lane < b.maxM0 ? links[lane] : EMPTY_LINK;
    const bool valid = link != EMPTY_LINK;
    const int cnt = __popc(__ballot_sync(FULL_MASK, valid));
    const uint8_t *xcode = b.node_codes + (size_t)x * M;
    if (cnt < b.maxM0) {
      if (lane == 0) links[cnt] = x;
      for (int t = lane; t < M; t += 32) codes[(size_t)cnt * M + t] = xcode[t];
    } else {
      uint8_t mycode[128];
      for (int t = 0; t < M; t++) mycode[t] = valid ? codes[(size_t)lane * M + t] : 0;
      float d = CUDART_INF_F;
      if (valid) d = adc_direct(q + (size_t)i * dim, cb, mycode, M, ds, is_ip, bias);
      const bool keep = valid && !(d < dr);
      int rank = 0;
      for (int s = 0; s < 32; s++) {
        const uint32_t oid = __shfl_sync(FULL_MASK, link, s);
        const bool ok = __shfl_sync(FULL_MASK, (int)keep, s);
        rank += (ok && oid > link) ? 1 : 0;
      }
      const int nkeep = __popc(__ballot_sync(FULL_MASK, keep));
      const int total = min(1 + nkeep, b.maxM0);
      __syncwarp();
      if (keep && 1 + rank < b.maxM0) {
        links[1 + rank] = link;
        for (int t = 0; t < M; t++) codes[(size_t)(1 + rank) * M + t] = mycode[t];
      }
      if (lane == 0) {
        links[0] = x;
        for (int t = 0; t < M; t++) codes[t] = xcode[t];
      }
      if (lane >= total && lane < b.maxM0) links[lane] = EMPTY_LINK;
    }
  }
}

// links of every node, maxM0 u32 each (0xFFFFFFFF = empty), for the host graph
__global__ void export_links_kernel(const uint8_t *__restrict__ rec0, int rec0_bytes, int maxM0, int64_t n, uint32_t *__restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * maxM0) return;
  const int64_t node = t / maxM0;
  const int j = (int)(t - node * maxM0);
  out[t] = reinterpret_cast<const uint32_t *>(rec0 + (size_t)node * rec0_bytes)[j];
}

// Phase 1 of a build: levels first (the index's own generator, in row order: what a sequential insertion would draw),
// then the rows that own upper-level lists + leading level-0 rows until the graph has a few thousand nodes, inserted on
// one host thread.  Row t of the batch is vectors + (rows ? rows[t] : t) * dim with label labels[t]; p2 receives the
// batch positions of the rows left for phase 2, in order.
int build_phase1(annb_index *h, const float *vectors, const int64_t *rows, const uint64_t *labels, int64_t n,
                 std::vector<int64_t> &p2) {
  HostGraph &g = h->g;
  const int dim = h->dim;
  const int64_t n_before = g.count.load();
  std::vector<int32_t> lv((size_t)n);
  ANNB_TRY_RC(hnsw_draw_levels(h, n, lv.data()));
  std::vector<int64_t> p1;
  const int64_t want = std::min<int64_t>(n, std::max<int64_t>(8192 - n_before, 1));
  int64_t lead = 0;
  for (int64_t i = 0; i < n; i++) {
    if (lv[i] > 0) p1.push_back(i);
    else if (lead < want) {
      p1.push_back(i);
      lead++;
    } else p2.push_back(i);
  }
  std::vector<float> v1(p1.size() * (size_t)dim);
  std::vector<uint64_t> l1(p1.size());
  std::vector<int32_t> f1(p1.size());
  for (size_t t = 0; t < p1.size(); t++) {
    memcpy(v1.data() + t * dim, vectors + (size_t)(rows ? rows[p1[t]] : p1[t]) * dim, (size_t)dim * 4);
    l1[t] = labels[p1[t]];
    f1[t] = lv[p1[t]];
  }
  // one thread: a concurrent host insertion would make the graph depend on thread timing (the build is deterministic)
  return hnsw_host_add(h, v1.data(), nullptr, l1.data(), (int64_t)p1.size(), 1, f1.data());
}

// The device graph of phase 1 with room for N nodes, and every node's own code (the first n1 uploaded) for phase 2
int build_device_graph(annb_index *h, int64_t N, BuildDev &b) {
  HostGraph &g = h->g;
  const int M = h->M;
  const int64_t n1 = g.count.load();
  h->dev_dirty = true;
  h->reserve_nodes = N;
  ANNB_TRY_RC(sync_device_graph(h));
  h->reserve_nodes = 0;
  b.rec0 = h->d_rec0;
  b.labels = h->d_labels;
  b.rec0_bytes = h->gd.rec0_bytes;
  b.code_off0 = h->gd.code_off0;
  b.maxM0 = g.maxM0;
  b.M = M;
  void *p;
  ANNB_TRY_RC(annb_scratch(h, S_RAW0, (size_t)N * M, &p));  // raw upload buffer is free again after the sync
  b.node_codes = (uint8_t *)p;
  std::vector<uint8_t> c1((size_t)n1 * M);
  for (int64_t i = 0; i < n1; i++) memcpy(c1.data() + (size_t)i * M, g.code((uint32_t)i), (size_t)M);
  ANNB_CUDA(cudaMemcpyAsync(b.node_codes, c1.data(), c1.size(), cudaMemcpyHostToDevice, h->stream));
  ANNB_CUDA(cudaStreamSynchronize(h->stream));
  return ANNB_OK;
}

// The host graph (nodes n1..N-1 new, labels l2[i - n1]) from the device records and node codes of phase 2
int build_finish(annb_index *h, const BuildDev &b, int64_t n1, int64_t N, const uint64_t *l2, int num_threads) {
  HostGraph &g = h->g;
  const int M = h->M;
  const int64_t n2 = N - n1;
  std::vector<uint32_t> hl((size_t)N * g.maxM0);
  std::vector<uint8_t> hc((size_t)n2 * M);
  {
    uint32_t *dl;
    ANNB_TRY_RC(annb_scratch(h, S_TOUCHED, hl.size() * 4, (void **)&dl));
    const int64_t tot = N * g.maxM0;
    export_links_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, h->stream>>>(b.rec0, b.rec0_bytes, g.maxM0, N, dl);
    ANNB_CUDA(cudaGetLastError());
    ANNB_CUDA(cudaMemcpyAsync(hl.data(), dl, hl.size() * 4, cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(hc.data(), b.node_codes + (size_t)n1 * M, hc.size(), cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
  }
  const int T = std::max(1, std::min(32, num_threads > 0 ? num_threads : 16));
  std::vector<std::thread> pool;
  for (int t = 0; t < T; t++) {
    pool.emplace_back([&, t] {
      for (int64_t i = N * t / T; i < N * (t + 1) / T; i++) {
        uint8_t *rec = g.rec0((uint32_t)i);
        if (i >= n1) {
          memset(rec, 0, g.size_per_elem);
          memcpy(rec + g.offset_data, hc.data() + (size_t)(i - n1) * M, (size_t)M);
          const uint64_t lab = l2[i - n1];
          memcpy(rec + g.label_offset, &lab, 8);
          g.levels[i] = 0;
        }
        const uint32_t *src = hl.data() + (size_t)i * g.maxM0;
        uint16_t cnt = 0;
        uint32_t *dst = reinterpret_cast<uint32_t *>(rec + 4);
        for (int j = 0; j < g.maxM0; j++)
          if (src[j] != EMPTY_LINK) dst[cnt++] = src[j];
        for (int j = cnt; j < g.maxM0; j++) dst[j] = 0;
        memcpy(rec, &cnt, 2);
      }
    });
  }
  for (auto &th : pool) th.join();
  g.label_lookup.reserve((size_t)N);
  for (int64_t i = n1; i < N; i++) g.label_lookup[l2[i - n1]] = (uint32_t)i;
  g.count.store(N);
  h->dev_dirty = true;  // the next search re-derives the device graph from the host graph: one source of truth
  return ANNB_OK;
}

}  // namespace

// gpu_build_run's geometry rule: the handle's level-0 records and codes are what phase 2's kernels cover
bool gpu_build_geometry(const annb_index *h) {
  const HostGraph &g = h->g;
  return h->Ks == 256 && h->code_bytes == 1 && (h->M == 8 || h->M == 16 || h->M == 32) && g.maxM0 <= 32 && g.maxM <= 32 &&
         h->d_codebook_t && h->cb_vec != 0 && g.num_deleted == 0 && g.M <= 32;
}

// Returns ANNB_OK, an error, or 1 = "not applicable here" (the caller then takes the host path).
int gpu_build_run(annb_index *h, const float *vectors, const uint64_t *labels, int64_t n, int num_threads) {
  HostGraph &g = h->g;
  if (n < 16384 || !gpu_build_geometry(h)) return 1;
  if (g.count.load() + n > g.max_elements) ANNB_FAIL(ANNB_ECAPACITY, "The number of elements exceeds the specified limit");
  for (int64_t i = 0; i < n; i++)
    if (g.label_lookup.find(labels[i]) != g.label_lookup.end()) return 1;  // updates of stored labels: host path
  {
    std::vector<uint64_t> s(labels, labels + n);
    std::sort(s.begin(), s.end());
    if (std::adjacent_find(s.begin(), s.end()) != s.end()) return 1;
  }
  const int M = h->M, dim = h->dim;
  std::vector<int64_t> p2;
  ANNB_TRY_RC(build_phase1(h, vectors, nullptr, labels, n, p2));
  const int64_t n1 = g.count.load();
  const int64_t n2 = (int64_t)p2.size();
  if (n2 == 0) {
    h->dev_dirty = true;
    return ANNB_OK;
  }
  const int64_t N = n1 + n2;

  // ---- device graph of phase 1, with room for everything ----------------------------------------------------
  BuildDev b;
  ANNB_TRY_RC(build_device_graph(h, N, b));

  // ---- phase 2 ----------------------------------------------------------------------------------------------
  const int k = g.M;
  const int ef = std::max(g.ef_construction, k);
  if (ef > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "ef_construction=%d exceeds ANNB_MAX_EF=%d", ef, ANNB_MAX_EF);
  const int64_t BMAX = 65536;
  float *dq;
  uint64_t *dsel, *dlab;
  float *dseld;
  int32_t *dfound;
  ANNB_TRY_RC(annb_scratch(h, S_QUERIES, (size_t)BMAX * dim * 4, (void **)&dq));
  ANNB_TRY_RC(annb_scratch(h, S_OUT_L, (size_t)BMAX * k * 8, (void **)&dsel));
  ANNB_TRY_RC(annb_scratch(h, S_OUT_D, (size_t)BMAX * k * 4, (void **)&dseld));
  ANNB_TRY_RC(annb_scratch(h, S_FOUND, (size_t)BMAX * 4, (void **)&dfound));
  ANNB_TRY_RC(annb_scratch(h, S_FLT_LABELS, (size_t)BMAX * 8, (void **)&dlab));
  float *hq;
  uint64_t *hlab;
  ANNB_TRY_RC(annb_pinned(h, 0, (size_t)BMAX * dim * 4, (void **)&hq));
  ANNB_TRY_RC(annb_pinned(h, 1, (size_t)BMAX * 8, (void **)&hlab));
  uint32_t *dcsr;  // a batch's back-links grouped by neighbour: [off (R+1)][rows (R)][pairs (P)]
  ANNB_TRY_RC(annb_scratch(h, S_CAND, ((size_t)3 * BMAX * k + 1) * 4, (void **)&dcsr));
  std::vector<uint64_t> hsel((size_t)BMAX * k);
  std::vector<int32_t> hfound((size_t)BMAX);
  std::vector<uint32_t> cnt((size_t)N), pos((size_t)N), hrows, hoff, hpairs;
  const int is_ip = h->metric != ANNB_METRIC_L2;
  const float bias = h->opt_ip_raw ? 0.f : (float)(1.0 / (double)h->Ks);
  int64_t n_cur = n1, done = 0;
  while (done < n2) {
    const int64_t B = std::min<int64_t>(n2 - done, std::max<int64_t>(256, std::min<int64_t>(BMAX, n_cur / std::max<int64_t>(1, h->opt_gpu_build_frac))));
    for (int64_t t = 0; t < B; t++) {
      memcpy(hq + (size_t)t * dim, vectors + (size_t)p2[done + t] * dim, (size_t)dim * 4);
      hlab[t] = labels[p2[done + t]];
    }
    ANNB_CUDA(cudaMemcpyAsync(dq, hq, (size_t)B * dim * 4, cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(dlab, hlab, (size_t)B * 8, cudaMemcpyHostToDevice, h->stream));
    // the reference encodes the row as handed in and builds its table from the re-normalised row (pq.py:309-310)
    ANNB_TRY_RC(launch_encode(h, dq, B, b.node_codes + (size_t)n_cur * M));
    if (h->metric == ANNB_METRIC_COSINE) ANNB_TRY_RC(launch_l2_normalize(h, dq, B, dim));
    SearchParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.queries = dq;
    sp.cbt = h->d_codebook_t;
    sp.cb_vec = h->cb_vec;
    sp.ds = h->ds;
    sp.is_ip = is_ip;
    sp.bias = bias;
    sp.B = B;
    sp.k = k;
    sp.ef = ef;
    sp.out_labels = dsel;
    sp.out_dists = dseld;
    sp.out_found = dfound;
    sp.out_internal = 1;
    int rc = launch_walk4(h, sp);
    if (rc == 1) ANNB_FAIL(ANNB_ESTATE, "internal: the search kernel does not cover this index");
    if (rc) return rc;
    const unsigned wb = 8;  // warps per block
    link_new_nodes_kernel<<<(unsigned)((B + wb - 1) / wb), wb * 32, 0, h->stream>>>(b, dsel, dfound, k, dlab, (uint32_t)n_cur, (int)B);
    // group the batch's (neighbour r, pair p) back-links by r, p ascending within each r (counting sort, stable)
    ANNB_CUDA(cudaMemcpyAsync(hsel.data(), dsel, (size_t)B * k * 8, cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(hfound.data(), dfound, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
    std::fill(cnt.begin(), cnt.begin() + n_cur, 0u);
    for (int64_t i = 0; i < B; i++)
      for (int j = 0; j < std::min(hfound[i], k); j++) {
        const uint64_t r = hsel[(size_t)i * k + j];
        if (r >= (uint64_t)n_cur) ANNB_FAIL(ANNB_ESTATE, "internal: GPU build selected node %llu of %lld", (unsigned long long)r, (long long)n_cur);
        cnt[r]++;
      }
    hrows.clear();
    hoff.clear();
    uint32_t acc = 0;
    for (int64_t r = 0; r < n_cur; r++)
      if (cnt[r]) {
        hrows.push_back((uint32_t)r);
        hoff.push_back(acc);
        pos[r] = acc;
        acc += cnt[r];
      }
    hoff.push_back(acc);
    hpairs.resize(acc);
    for (int64_t i = 0; i < B; i++)
      for (int j = 0; j < std::min(hfound[i], k); j++) hpairs[pos[hsel[(size_t)i * k + j]]++] = (uint32_t)(i * k + j);
    const int R = (int)hrows.size();
    ANNB_CUDA(cudaMemcpyAsync(dcsr, hoff.data(), hoff.size() * 4, cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(dcsr + R + 1, hrows.data(), hrows.size() * 4, cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaMemcpyAsync(dcsr + 2 * R + 1, hpairs.data(), hpairs.size() * 4, cudaMemcpyHostToDevice, h->stream));
    if (R > 0)
      reverse_link_kernel<<<(unsigned)((R + wb - 1) / wb), wb * 32, 0, h->stream>>>(b, dcsr + R + 1, dcsr, dcsr + 2 * R + 1, R, dseld, k, dq, dim,
                                                                                    h->d_codebook, h->ds, is_ip, bias, (uint32_t)n_cur);
    h->launches += 2;
    ANNB_CUDA(cudaGetLastError());
    ANNB_CUDA(cudaStreamSynchronize(h->stream));  // hq / hlab are refilled next
    n_cur += B;
    done += B;
    h->gd.n = n_cur;
  }

  // ---- host graph from the device records --------------------------------------------------------------------
  std::vector<uint64_t> l2((size_t)n2);
  for (int64_t i = 0; i < n2; i++) l2[i] = labels[p2[i]];
  return build_finish(h, b, n1, N, l2.data(), num_threads);
}

// ---- a cell-set insertion (annb_cellset_add_items) ---------------------------------------------------------------
namespace {

// a device / pinned buffer that grows on demand (contents are not kept)
struct GrowBuf {
  void *p = nullptr;
  size_t cap = 0;
  bool pinned = false;
  explicit GrowBuf(bool pinned_ = false) : pinned(pinned_) {}
  ~GrowBuf() {
    if (p) pinned ? cudaFreeHost(p) : cudaFree(p);  // both wait for the work using the buffer
  }
  int get(size_t bytes, void **out) {
    if (bytes == 0) bytes = 16;
    if (cap < bytes) {
      if (p) pinned ? cudaFreeHost(p) : cudaFree(p);
      p = nullptr;
      cap = 0;
      const size_t c = (bytes + bytes / 4 + 255) / 256 * 256;
      if ((pinned ? cudaMallocHost(&p, c) : cudaMalloc(&p, c)) != cudaSuccess) {
        cudaGetLastError();
        p = nullptr;
        ANNB_FAIL(ANNB_ENOMEM, "%s(%zu bytes) failed", pinned ? "cudaMallocHost" : "cudaMalloc", c);
      }
      cap = c;
    }
    *out = p;
    return ANNB_OK;
  }
};

struct CellBuildState {
  std::vector<int64_t> p2;  // positions (in the job's rows) of the rows phase 2 inserts
  int64_t n1 = 0, N = 0, n_cur = 0, done = 0;
  int k = 0, ef = 0;
  BuildDev b{};
  std::vector<uint32_t> cnt, pos;  // the counting sort of a round's back-links by neighbour
  int rc = ANNB_OK;
  std::string err;
};

int cell_ef(const annb_index *h) { return std::max(h->g.ef_construction, h->g.M); }

// phase 1 of one cell and its device graph with room for every row (runs on the cell's own thread and stream)
int cell_phase1(CellBuildJob &j, CellBuildState &s) {
  annb_index *h = j.h;
  ANNB_CUDA(cudaSetDevice(h->device));
  ANNB_TRY_RC(build_phase1(h, j.vectors, j.rows.data(), j.labels.data(), (int64_t)j.rows.size(), s.p2));
  s.n1 = s.n_cur = h->g.count.load();
  s.N = s.n1 + (int64_t)s.p2.size();
  if (s.p2.empty()) {
    h->dev_dirty = true;
    return ANNB_OK;
  }
  s.k = h->g.M;
  s.ef = cell_ef(h);
  if (s.ef > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "ef_construction=%d exceeds ANNB_MAX_EF=%d", s.ef, ANNB_MAX_EF);
  ANNB_TRY_RC(build_device_graph(h, s.N, s.b));
  s.cnt.assign((size_t)s.N, 0u);
  s.pos.resize((size_t)s.N);
  return ANNB_OK;
}

// a walk launch of a round: cells [e0, e1) (one ef), their rows [r0, r0 + rows) of the round
struct BuildGroup {
  int e0 = 0, e1 = 0, kmax = 0;
  int64_t r0 = 0, rows = 0;
};

constexpr int64_t BUILD_BMAX = 65536;                  // gpu_build_run's largest batch
constexpr size_t BUILD_SCRATCH_CAP = (size_t)256 << 20; // by-cell scratch of one walk launch: (rows, cells, kmax) x 12 B

}  // namespace

int gpu_build_cells(annb_index *drv, std::vector<CellBuildJob> &jobs, int num_threads, CellBuildStats *stats) {
  const int E = (int)jobs.size();
  if (E == 0) return ANNB_OK;
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  // cells with the same ef are neighbours in the descriptor array: one walk launch can serve a run of them
  std::stable_sort(jobs.begin(), jobs.end(), [](const CellBuildJob &a, const CellBuildJob &b) { return cell_ef(a.h) < cell_ef(b.h); });
  std::vector<CellBuildState> cs((size_t)E);

  // ---- phase 1, one host thread per cell at a time (cells share no state; each stays deterministic) ---------------
  {
    const int T = std::max(1, std::min<int>(E, (int)std::max(1u, std::thread::hardware_concurrency())));
    std::atomic<int> next{0};
    std::vector<std::thread> pool;
    for (int t = 0; t < T; t++)
      pool.emplace_back([&] {
        for (int e = next++; e < E; e = next++) {
          cs[e].rc = cell_phase1(jobs[e], cs[e]);
          if (cs[e].rc) cs[e].err = annb_last_error();
        }
      });
    for (auto &th : pool) th.join();
  }
  ANNB_CUDA(cudaSetDevice(drv->device));
  for (int e = 0; e < E; e++)
    if (cs[e].rc) ANNB_FAIL(cs[e].rc, "cell %d: %s", jobs[e].cell, cs[e].err.c_str());
  const auto t1 = clk::now();

  // ---- phase 2 in rounds: every cell's next batch, each searching its own graph as it stood before the round ------
  cudaStream_t st = drv->stream;
  const int dim = drv->dim, M = drv->M;
  const int is_ip = drv->metric != ANNB_METRIC_L2;
  const float bias = drv->opt_ip_raw ? 0.f : (float)(1.0 / (double)drv->Ks);
  GrowBuf d_bd, d_gd, d_ck, d_q, d_lab, d_rc, d_rn, d_sl, d_sd, d_sf, d_csr;
  GrowBuf h_q(true), h_lab(true), h_rc(true), h_rn(true);
  BuildDev *bd;
  GraphDev *gd;
  int32_t *ck;
  ANNB_TRY_RC(d_bd.get((size_t)E * sizeof(BuildDev), (void **)&bd));
  ANNB_TRY_RC(d_gd.get((size_t)E * sizeof(GraphDev), (void **)&gd));
  ANNB_TRY_RC(d_ck.get((size_t)E * 4, (void **)&ck));
  std::vector<BuildDev> bdh((size_t)E);
  std::vector<GraphDev> gdh((size_t)E);
  std::vector<int32_t> ckh((size_t)E);
  for (int e = 0; e < E; e++) {
    bdh[e] = cs[e].b;
    ckh[e] = cs[e].k;
  }
  ANNB_CUDA(cudaMemcpyAsync(bd, bdh.data(), bdh.size() * sizeof(BuildDev), cudaMemcpyHostToDevice, st));
  ANNB_CUDA(cudaMemcpyAsync(ck, ckh.data(), ckh.size() * 4, cudaMemcpyHostToDevice, st));
  std::vector<int64_t> Bc((size_t)E), off((size_t)E);
  std::vector<BuildGroup> groups;
  std::vector<uint64_t> hsel;
  std::vector<int32_t> hfound, hrcell;
  std::vector<uint32_t> hrows, hoff, hpairs;
  int64_t rounds = 0;
  for (;;) {
    // each cell's batch is the one gpu_build_run picks from that cell's own n_cur
    int64_t R = 0;
    for (int e = 0; e < E; e++) {
      const CellBuildState &s = cs[e];
      const int64_t n2 = (int64_t)s.p2.size(), frac = std::max<int64_t>(1, jobs[e].h->opt_gpu_build_frac);
      Bc[e] = s.done < n2 ? std::min<int64_t>(n2 - s.done, std::max<int64_t>(256, std::min<int64_t>(BUILD_BMAX, s.n_cur / frac))) : 0;
      off[e] = R;
      R += Bc[e];
    }
    if (R == 0) break;
    rounds++;
    groups.clear();
    for (int e = 0; e < E; e++) {
      if (!Bc[e]) continue;
      BuildGroup *g = groups.empty() ? nullptr : &groups.back();
      const int kmax = g ? std::max(g->kmax, cs[e].k) : cs[e].k;
      if (!g || cs[g->e0].ef != cs[e].ef ||
          (size_t)(g->rows + Bc[e]) * (size_t)(e + 1 - g->e0) * (size_t)kmax * 12 > BUILD_SCRATCH_CAP) {
        BuildGroup ng;
        ng.e0 = e;
        ng.r0 = off[e];
        groups.push_back(ng);
        g = &groups.back();
      }
      g->e1 = e + 1;
      g->rows += Bc[e];
      g->kmax = std::max(g->kmax, cs[e].k);
    }
    // the round's rows, labels, cells (local to the row's launch) and node ids
    float *hq, *dq;
    uint64_t *hlab, *dlab;
    int32_t *hrc, *drc;
    uint32_t *hrn, *drn;
    ANNB_TRY_RC(h_q.get((size_t)R * dim * 4, (void **)&hq));
    ANNB_TRY_RC(h_lab.get((size_t)R * 8, (void **)&hlab));
    ANNB_TRY_RC(h_rc.get((size_t)R * 4, (void **)&hrc));
    ANNB_TRY_RC(h_rn.get((size_t)R * 4, (void **)&hrn));
    ANNB_TRY_RC(d_q.get((size_t)R * dim * 4, (void **)&dq));
    ANNB_TRY_RC(d_lab.get((size_t)R * 8, (void **)&dlab));
    ANNB_TRY_RC(d_rc.get((size_t)R * 4, (void **)&drc));
    ANNB_TRY_RC(d_rn.get((size_t)R * 4, (void **)&drn));
    for (const BuildGroup &g : groups)
      for (int e = g.e0; e < g.e1; e++) {
        const CellBuildJob &j = jobs[e];
        const CellBuildState &s = cs[e];
        for (int64_t t = 0; t < Bc[e]; t++) {
          const int64_t at = s.p2[s.done + t], r = off[e] + t;
          memcpy(hq + (size_t)r * dim, j.vectors + (size_t)j.rows[at] * dim, (size_t)dim * 4);
          hlab[r] = j.labels[at];
          hrc[r] = e - g.e0;
          hrn[r] = (uint32_t)(s.n_cur + t);
        }
      }
    ANNB_CUDA(cudaMemcpyAsync(dq, hq, (size_t)R * dim * 4, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(dlab, hlab, (size_t)R * 8, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(drc, hrc, (size_t)R * 4, cudaMemcpyHostToDevice, st));
    ANNB_CUDA(cudaMemcpyAsync(drn, hrn, (size_t)R * 4, cudaMemcpyHostToDevice, st));
    // encode each cell's segment into its node codes (the cells share the codebook), then normalise once for cosine:
    // the reference encodes the row as handed in and builds its table from the re-normalised row (pq.py:309-310)
    for (int e = 0; e < E; e++)
      if (Bc[e]) ANNB_TRY_RC(launch_encode(drv, dq + (size_t)off[e] * dim, Bc[e], cs[e].b.node_codes + (size_t)cs[e].n_cur * M));
    if (drv->metric == ANNB_METRIC_COSINE) ANNB_TRY_RC(launch_l2_normalize(drv, dq, R, dim));
    for (int e = 0; e < E; e++) {
      gdh[e] = jobs[e].h->gd;
      gdh[e].n = cs[e].n_cur;
    }
    ANNB_CUDA(cudaMemcpyAsync(gd, gdh.data(), gdh.size() * sizeof(GraphDev), cudaMemcpyHostToDevice, st));

    for (const BuildGroup &g : groups) {
      const int span = g.e1 - g.e0, kmax = g.kmax;
      const size_t slots = (size_t)g.rows * span;
      uint64_t *sl;
      float *sd;
      int32_t *sf;
      ANNB_TRY_RC(d_sl.get(slots * kmax * 8, (void **)&sl));
      ANNB_TRY_RC(d_sd.get(slots * kmax * 4, (void **)&sd));
      ANNB_TRY_RC(d_sf.get(slots * 4, (void **)&sf));
      // construction search: each row probes its own cell only, k = that cell's M_, internal ids out
      SearchParams sp;
      memset(&sp, 0, sizeof(sp));
      sp.queries = dq + (size_t)g.r0 * dim;
      sp.cbt = drv->d_codebook_t;
      sp.cb_vec = drv->cb_vec;
      sp.ds = drv->ds;
      sp.is_ip = is_ip;
      sp.bias = bias;
      sp.B = g.rows;
      sp.k = kmax;
      sp.ef = cs[g.e0].ef;
      sp.out_labels = sl;
      sp.out_dists = sd;
      sp.out_found = sf;
      sp.out_internal = 1;
      sp.cells = gd + g.e0;
      sp.cell_order = drc + g.r0;
      sp.cell_k = ck + g.e0;
      sp.n_cells = span;
      sp.n_probe = 1;
      sp.cell_limit = kmax;
      const int rc = launch_walk4_cells(drv, sp);
      if (rc == 1) ANNB_FAIL(ANNB_ESTATE, "internal: the multi-cell walk does not cover these cells");
      if (rc) return rc;
      const unsigned wb = 8;  // warps per block
      link_new_nodes_cells_kernel<<<(unsigned)((g.rows + wb - 1) / wb), wb * 32, 0, st>>>(
          bd + g.e0, ck + g.e0, drc + g.r0, drn + g.r0, sl, sf, span, kmax, dlab + g.r0, (int)g.rows);
      ANNB_CUDA(cudaGetLastError());
      // each cell segment's candidates back for the counting sort
      hsel.resize((size_t)g.rows * kmax);
      hfound.resize((size_t)g.rows);
      for (int e = g.e0; e < g.e1; e++) {
        if (!Bc[e]) continue;
        const int64_t a = off[e] - g.r0;
        const int c = e - g.e0;
        ANNB_CUDA(cudaMemcpy2DAsync(hsel.data() + (size_t)a * kmax, (size_t)kmax * 8, sl + ((size_t)a * span + c) * kmax,
                                    (size_t)span * kmax * 8, (size_t)cs[e].k * 8, (size_t)Bc[e], cudaMemcpyDeviceToHost, st));
        ANNB_CUDA(cudaMemcpy2DAsync(hfound.data() + a, 4, sf + (size_t)a * span + c, (size_t)span * 4, 4, (size_t)Bc[e],
                                    cudaMemcpyDeviceToHost, st));
      }
      ANNB_CUDA(cudaStreamSynchronize(st));
      // per cell, the back-links grouped by neighbour r, pair order within r (gpu_build_run's counting sort)
      hrows.clear();
      hrcell.clear();
      hoff.clear();
      uint32_t acc = 0;
      for (int e = g.e0; e < g.e1; e++) {
        if (!Bc[e]) continue;
        CellBuildState &s = cs[e];
        const int64_t a = off[e] - g.r0;
        const int k = s.k;
        std::fill(s.cnt.begin(), s.cnt.begin() + s.n_cur, 0u);
        for (int64_t i = a; i < a + Bc[e]; i++)
          for (int j = 0; j < std::min(hfound[i], k); j++) {
            const uint64_t r = hsel[(size_t)i * kmax + j];
            if (r >= (uint64_t)s.n_cur)
              ANNB_FAIL(ANNB_ESTATE, "cell %d: internal: GPU build selected node %llu of %lld", jobs[e].cell, (unsigned long long)r,
                        (long long)s.n_cur);
            s.cnt[r]++;
          }
        for (int64_t r = 0; r < s.n_cur; r++)
          if (s.cnt[r]) {
            hrows.push_back((uint32_t)r);
            hrcell.push_back(e - g.e0);
            hoff.push_back(acc);
            s.pos[r] = acc;
            acc += s.cnt[r];
          }
        hpairs.resize(acc);
        for (int64_t i = a; i < a + Bc[e]; i++)
          for (int j = 0; j < std::min(hfound[i], k); j++) hpairs[s.pos[hsel[(size_t)i * kmax + j]]++] = (uint32_t)(i * kmax + j);
      }
      hoff.push_back(acc);
      const int Rn = (int)hrows.size();
      uint32_t *csr;  // [off (Rn+1)][rows (Rn)][cells (Rn)][pairs (acc)]
      ANNB_TRY_RC(d_csr.get(((size_t)3 * Rn + 1 + acc) * 4, (void **)&csr));
      ANNB_CUDA(cudaMemcpyAsync(csr, hoff.data(), hoff.size() * 4, cudaMemcpyHostToDevice, st));
      ANNB_CUDA(cudaMemcpyAsync(csr + Rn + 1, hrows.data(), hrows.size() * 4, cudaMemcpyHostToDevice, st));
      ANNB_CUDA(cudaMemcpyAsync(csr + 2 * Rn + 1, hrcell.data(), hrcell.size() * 4, cudaMemcpyHostToDevice, st));
      ANNB_CUDA(cudaMemcpyAsync(csr + 3 * Rn + 1, hpairs.data(), (size_t)acc * 4, cudaMemcpyHostToDevice, st));
      if (Rn > 0)
        reverse_link_cells_kernel<<<(unsigned)((Rn + wb - 1) / wb), wb * 32, 0, st>>>(
            bd + g.e0, reinterpret_cast<const int32_t *>(csr + 2 * Rn + 1), csr + Rn + 1, csr, csr + 3 * Rn + 1, Rn, sd, drn + g.r0,
            span, kmax, dq + (size_t)g.r0 * dim, dim, drv->d_codebook, drv->ds, is_ip, bias);
      drv->launches += 2;
      ANNB_CUDA(cudaGetLastError());
    }
    ANNB_CUDA(cudaStreamSynchronize(st));  // the pinned rows are refilled next round
    for (int e = 0; e < E; e++) {
      cs[e].n_cur += Bc[e];
      cs[e].done += Bc[e];
      jobs[e].h->gd.n = cs[e].n_cur;
    }
  }

  // ---- each host graph from its device records --------------------------------------------------------------------
  for (int e = 0; e < E; e++) {
    CellBuildState &s = cs[e];
    if (s.p2.empty()) continue;
    std::vector<uint64_t> l2(s.p2.size());
    for (size_t i = 0; i < s.p2.size(); i++) l2[i] = jobs[e].labels[s.p2[i]];
    const int rc = build_finish(jobs[e].h, s.b, s.n1, s.N, l2.data(), num_threads);
    if (rc) {
      const std::string msg = annb_last_error();
      ANNB_FAIL(rc, "cell %d: %s", jobs[e].cell, msg.c_str());
    }
  }
  if (stats) {
    stats->phase1_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    stats->phase2_ms = std::chrono::duration<double, std::milli>(clk::now() - t1).count();
    stats->rounds = rounds;
  }
  return ANNB_OK;
}
