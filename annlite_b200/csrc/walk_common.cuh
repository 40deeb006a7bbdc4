// walk_common.cuh -- pieces shared by the warp-per-query walks: the persistent loop's work counter, the result row
// epilogue of the WarpList walks (hnsw_search.cu, walk_wide.cu), the tie fix-up every walk's epilogue runs, and the
// host loop that runs a bitmap walk (hnsw_walk_general, hnsw_walk_wide) with its per-warp scratch.
#pragma once
#include <math_constants.h>

#include <algorithm>

#include "annb_internal.h"
#include "warp_list.cuh"

namespace {

constexpr uint32_t EMPTY_LINK = 0xffffffffu;
constexpr uint32_t ID_MASK = 0x7fffffffu;
constexpr int SBAG = 256;  // candidate bag entries kept in shared memory per warp (spills to global beyond)

// Next query of the persistent loop: ONE lane bumps the work counter (a predicated instruction, not a branch) and
// the value is spread with a warp REDUCTION: REDUX delivers it in a uniform register, so ptxas can prove that the
// loop exit is warp-uniform.  With `__shfl_sync(qi, 0)` it cannot, and then guards every warp-level operation of the
// loop body with a BRA.DIV convergence check.
__device__ __forceinline__ int64_t next_query(unsigned int *counter, int lane) {
  unsigned qi = 0;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.eq.u32 p, %2, 0;\n"
      "@p atom.global.add.u32 %0, [%1], 1;\n"
      "}\n"
      : "+r"(qi)
      : "l"(counter), "r"(lane)
      : "memory");
  return (int64_t)__reduce_max_sync(FULL_MASK, qi);
}

// candidate bag entry of the bitmap walks
__device__ __forceinline__ uint64_t pack_cand(float d, uint32_t id) { return ((uint64_t)__float_as_uint(d) << 32) | id; }
__device__ __forceinline__ float cand_d(uint64_t c) { return __uint_as_float((uint32_t)(c >> 32)); }
__device__ __forceinline__ uint32_t cand_id(uint64_t c) { return (uint32_t)c; }

// Rows must be ascending by (dist, label) (hnsw_bindings.cpp:346-351); a walk's list orders equal distances by arrival.
// One lane insertion-sorts the first `found` entries of the output row that starts at entry `row`; equal distances are
// rare, so it runs only after a tie.  The output arrays are read through the kernel parameters at each use, so they
// take no registers in the walk (copies in registers change the walks' register allocation).
__device__ __forceinline__ void sort_ties(const SearchParams &p, int64_t row, int found) {
  for (int i = 1; i < found; i++) {
    const float d = p.out_dists[row + i];
    const uint64_t l = p.out_labels[row + i];
    int j = i - 1;
    while (j >= 0 && p.out_dists[row + j] == d && p.out_labels[row + j] > l) {
      p.out_dists[row + j + 1] = p.out_dists[row + j];
      p.out_labels[row + j + 1] = p.out_labels[row + j];
      j--;
    }
    p.out_dists[row + j + 1] = d;
    p.out_labels[row + j + 1] = l;
  }
}

template <int EPL>
__device__ __forceinline__ void write_results(const GraphDev &g, const SearchParams &p, int64_t q, const WarpList<EPL> &L,
                                              int lane, int hops, int nbrs, int evals) {
  const int k = p.k;
  bool tie = false;
  int found = 0;
#pragma unroll
  for (int e = 0; e < EPL; e++) {
    const int pos = e * 32 + lane;
    const bool have = L.v[e] != LIST_EMPTY_VAL && pos < k;
    found += __popc(__ballot_sync(FULL_MASK, have));
    // tie detection between adjacent list positions
    float nk = __shfl_down_sync(FULL_MASK, L.k[e], 1);
    const float first_next = (e + 1 < EPL) ? __shfl_sync(FULL_MASK, L.k[(e + 1 < EPL) ? e + 1 : e], 0) : CUDART_INF_F;
    if (lane == 31) nk = first_next;
    tie |= have && (pos + 1 < k) && (nk == L.k[e]);
    if (pos < k) {
      p.out_dists[q * k + pos] = have ? L.k[e] : CUDART_INF_F;
      p.out_labels[q * k + pos] = have ? __ldg(g.labels + (L.v[e] & ID_MASK)) : (uint64_t)UINT64_MAX;
    }
  }
  tie = __any_sync(FULL_MASK, tie);
  if (tie) {
    __syncwarp();
    if (lane == 0) sort_ties(p, q * k, found);
  }
  if (lane == 0) {
    p.out_found[q] = found;
    if (p.out_stats) {
      p.out_stats[q * 3 + 0] = hops;
      p.out_stats[q * 3 + 1] = nbrs;
      p.out_stats[q * 3 + 2] = evals;
    }
  }
}

// Runs a bitmap walk on `blocks` CTAs of `warps` warps with its per-warp scratch: visited bitmaps (scratch slot 5),
// visited log (slot 6) and candidate bag (slot 7).  launch(blocks, p) enqueues one attempt on h->stream; p.work_counter
// is already zeroed for the first.  The log and the bag start at sizes that cover ordinary filters and grow (x4, up to
// the node count: neither can hold more) while a query outgrows them -- a very selective filter or many deletions make
// the walk visit a large part of the graph, as the reference's does.  `walk` names the walk in the overflow error.
template <typename Launch>
int run_bitmap_walk(annb_index *h, SearchParams &p, int blocks, int warps, const char *walk, Launch launch) {
  p.visited_words = (h->gd.n + 31) / 32;
  const int64_t cap_max = std::max<int64_t>(1 << 15, h->gd.n + 64);
  int64_t tcap = 1 << 15, ccap = 1 << 14;
  for (;;) {
    p.touched_cap = (int)std::min<int64_t>(tcap, cap_max);
    p.cand_cap = (int)std::min<int64_t>(ccap, cap_max);
    // keep the per-warp scratch within ~8 GB: fewer resident warps when each needs a lot
    while (blocks > 1 && (double)blocks * warps * ((double)p.touched_cap * 4 + (double)p.cand_cap * 8) > 8e9) blocks /= 2;
    const int64_t slots = (int64_t)blocks * warps;
    // every query leaves its visited bitmap all-zero, so the bitmaps are cleared only when (re)allocated
    const size_t before = h->scratch_cap[5];
    ANNB_TRY_RC(annb_scratch(h, 5, (size_t)slots * p.visited_words * 4, (void **)&p.visited));
    if (h->scratch_cap[5] != before) ANNB_CUDA(cudaMemsetAsync(p.visited, 0, h->scratch_cap[5], h->stream));
    ANNB_TRY_RC(annb_scratch(h, 6, (size_t)slots * p.touched_cap * 4, (void **)&p.touched));
    ANNB_TRY_RC(annb_scratch(h, 7, (size_t)slots * p.cand_cap * 8, (void **)&p.cand));
    launch(blocks, p);
    h->launches++;
    ANNB_CUDA(cudaGetLastError());
    int32_t flag = 0;
    ANNB_CUDA(cudaMemcpyAsync(&flag, p.overflow_flag, 4, cudaMemcpyDeviceToHost, h->stream));
    ANNB_CUDA(cudaStreamSynchronize(h->stream));
    if (!flag) return ANNB_OK;
    // visited bitmaps may be dirty after an overflow: wipe, then retry with more room
    ANNB_CUDA(cudaMemsetAsync(h->d_scratch[5], 0, h->scratch_cap[5], h->stream));
    if (p.touched_cap >= cap_max && p.cand_cap >= cap_max)
      ANNB_FAIL(ANNB_ELIMIT, "%s walk scratch overflow (candidate bag %d / visited log %d entries per query)", walk, p.cand_cap,
                p.touched_cap);
    ANNB_CUDA(cudaMemsetAsync(p.work_counter, 0, 8, h->stream));  // the counter and the overflow flag
    tcap *= 4;
    ccap *= 4;
  }
}

}  // namespace
