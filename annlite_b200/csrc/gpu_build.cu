// gpu_build.cu -- batched HNSW insertion with the level-0 work on the GPU (SURVEY.md section 8f, rank 2, second half).
//
// Reference: addPoint (include/hnswlib/hnswalg.h:1108-1235) = greedy descent, then per level searchBaseLayer at
// ef_construction (:158-238), getNeighborsByHeuristic2 (:443-483) and mutuallyConnectNewElement (:502-619).  In PQ
// mode the reference's "distance between two stored nodes" is the distance from the point being inserted to the
// second node (PQLookup ignores its first argument, SURVEY.md section 0.2), which collapses the heuristic:
//   * the new node x links to the M_ nearest of its ef_construction candidates, farthest first;
//   * a selected neighbour r with room appends x; a full one keeps x and those of its neighbours that are NOT
//     closer to x than r itself is (in descending id order, at most maxM0 of them).
// hnsw_build.cpp restates that on the host, byte for byte.  Here the same rules run batch-wise on the device:
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
// The graph is NOT the one a sequential build makes; what is checked is what matters for the path: every structural
// invariant (HostGraph::validate), oracle parity of searches over the result, and recall against a host-built
// graph of the same data (tests/test_gpu_build.py).
#include <math_constants.h>

#include <algorithm>
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

// links of every node, maxM0 u32 each (0xFFFFFFFF = empty), for the host graph
__global__ void export_links_kernel(const uint8_t *__restrict__ rec0, int rec0_bytes, int maxM0, int64_t n, uint32_t *__restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * maxM0) return;
  const int64_t node = t / maxM0;
  const int j = (int)(t - node * maxM0);
  out[t] = reinterpret_cast<const uint32_t *>(rec0 + (size_t)node * rec0_bytes)[j];
}

}  // namespace

// Returns ANNB_OK, an error, or 1 = "not applicable here" (the caller then takes the host path).
int gpu_build_run(annb_index *h, const float *vectors, const uint64_t *labels, int64_t n, int num_threads) {
  HostGraph &g = h->g;
  if (n < 16384 || h->Ks != 256 || h->code_bytes != 1 || !(h->M == 8 || h->M == 16 || h->M == 32) || g.maxM0 > 32 || g.maxM > 32 ||
      !h->d_codebook_t || h->cb_vec == 0 || g.num_deleted > 0 || g.M > 32)
    return 1;
  if (g.count.load() + n > g.max_elements) ANNB_FAIL(ANNB_ECAPACITY, "The number of elements exceeds the specified limit");
  for (int64_t i = 0; i < n; i++)
    if (g.label_lookup.find(labels[i]) != g.label_lookup.end()) return 1;  // updates of stored labels: host path
  {
    std::vector<uint64_t> s(labels, labels + n);
    std::sort(s.begin(), s.end());
    if (std::adjacent_find(s.begin(), s.end()) != s.end()) return 1;
  }
  const int M = h->M, dim = h->dim;
  const int64_t n_before = g.count.load();

  // ---- levels first (the index's own generator, in row order: what a sequential insertion would draw) ----------
  std::vector<int32_t> lv((size_t)n);
  ANNB_TRY_RC(hnsw_draw_levels(h, n, lv.data()));
  // phase 1 = rows that own upper-level lists + leading level-0 rows until the graph has a few thousand nodes
  std::vector<int64_t> p1, p2;
  const int64_t want = std::min<int64_t>(n, std::max<int64_t>(8192 - n_before, 1));
  int64_t lead = 0;
  for (int64_t i = 0; i < n; i++) {
    if (lv[i] > 0) p1.push_back(i);
    else if (lead < want) {
      p1.push_back(i);
      lead++;
    } else p2.push_back(i);
  }
  {
    std::vector<float> v1(p1.size() * (size_t)dim);
    std::vector<uint64_t> l1(p1.size());
    std::vector<int32_t> f1(p1.size());
    for (size_t t = 0; t < p1.size(); t++) {
      memcpy(v1.data() + t * dim, vectors + (size_t)p1[t] * dim, (size_t)dim * 4);
      l1[t] = labels[p1[t]];
      f1[t] = lv[p1[t]];
    }
    // one thread: a concurrent host insertion would make the graph depend on thread timing (the build is deterministic)
    ANNB_TRY_RC(hnsw_host_add(h, v1.data(), nullptr, l1.data(), (int64_t)p1.size(), 1, f1.data()));
  }
  const int64_t n1 = g.count.load();
  const int64_t n2 = (int64_t)p2.size();
  if (n2 == 0) {
    h->dev_dirty = true;
    return ANNB_OK;
  }
  const int64_t N = n1 + n2;

  // ---- device graph of phase 1, with room for everything ----------------------------------------------------
  h->dev_dirty = true;
  h->reserve_nodes = N;
  ANNB_TRY_RC(sync_device_graph(h));
  h->reserve_nodes = 0;
  BuildDev b;
  b.rec0 = h->d_rec0;
  b.labels = h->d_labels;
  b.rec0_bytes = h->gd.rec0_bytes;
  b.code_off0 = h->gd.code_off0;
  b.maxM0 = g.maxM0;
  b.M = M;
  void *p;
  ANNB_TRY_RC(annb_scratch(h, S_RAW0, (size_t)N * M, &p));  // raw upload buffer is free again after the sync
  b.node_codes = (uint8_t *)p;
  {
    std::vector<uint8_t> c1((size_t)n1 * M);
    for (int64_t i = 0; i < n1; i++) memcpy(c1.data() + (size_t)i * M, g.code((uint32_t)i), (size_t)M);
    ANNB_CUDA(cudaMemcpyAsync(b.node_codes, c1.data(), c1.size(), cudaMemcpyHostToDevice, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
  }

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
          const uint64_t lab = labels[p2[i - n1]];
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
  for (int64_t i = n1; i < N; i++) g.label_lookup[labels[p2[i - n1]]] = (uint32_t)i;
  g.count.store(N);
  h->dev_dirty = true;  // the next search re-derives the device graph from the host graph: one source of truth
  return ANNB_OK;
}
