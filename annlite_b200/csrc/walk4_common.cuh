// walk4_common.cuh -- pieces shared by hnsw_walk4 (walk_fused.cu) and hnsw_walk4f (walk_flagged4.cu): the
// order-preserving key image, a level-0 record in registers, the PQ lookup with compile-time M and Ks = 256, the
// register-resident sorted list (blocked: lane l holds positions l*EPL .. l*EPL+EPL-1) and the in-shared-memory
// ADC table build (K1 inside the walk), the CTA shape of both kernels and their launch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <type_traits>

#include "annb_internal.h"
#include "walk_common.cuh"

namespace {

constexpr uint32_t EXP_BIT = 0x80000000u;   // list value: node already expanded (empty slots carry it too)
constexpr uint32_t IDM = 0x7fffffffu;
constexpr uint32_t KEY_MAX = 0xffffffffu;   // above the image of every finite distance and of +inf

// order-preserving map fp32 -> u32 (a < b  <=>  f2u(a) < f2u(b) for non-NaN, no -0.0: the ADC sum starts
// at +0.f and x + (-0) never yields -0)
__device__ __forceinline__ uint32_t f2u(float f) {
  const uint32_t b = __float_as_uint(f);
  return b ^ ((uint32_t)((int32_t)b >> 31) | 0x80000000u);
}
__device__ __forceinline__ float u2f(uint32_t u) {
  return __uint_as_float(u ^ (((u >> 31) - 1u) | 0x80000000u));
}

// ---- one level-0 record in registers: lane j holds link j and the M code bytes of neighbour j ----
template <int M>
struct Rec {
  uint32_t link;
  uint32_t cw[M / 4];
};

template <int M>
__device__ __forceinline__ void load_codes(uint32_t (&cw)[M / 4], const uint8_t *p) {
  if (M == 4) {
    cw[0] = __ldg(reinterpret_cast<const uint32_t *>(p));
  } else if (M == 8) {
    const uint2 t = __ldg(reinterpret_cast<const uint2 *>(p));
    cw[0] = t.x;
    cw[1] = t.y;
  } else {
#pragma unroll
    for (int i = 0; i < M / 16; i++) {
      const uint4 t = __ldg(reinterpret_cast<const uint4 *>(p) + i);
      cw[4 * i + 0] = t.x;
      cw[4 * i + 1] = t.y;
      cw[4 * i + 2] = t.z;
      cw[4 * i + 3] = t.w;
    }
  }
}

// PQLookup (space_pq.h:30-35): strictly sequential fp32 sum over the M subquantisers, from 0.f
template <int M>
__device__ __forceinline__ float pq_score(const float *T, const uint32_t (&cw)[M / 4]) {
  float r = 0.f;
#pragma unroll
  for (int m = 0; m < M; m++) {
    const uint32_t code = (cw[m >> 2] >> (8 * (m & 3))) & 0xffu;
    r = __fadd_rn(r, T[m * 256 + code]);
  }
  return r;
}

// ---- the list: EPL entries per lane, position p = lane*EPL + e, ascending keys, dense from 0 ----
template <int EPL>
__device__ __forceinline__ void list_insert(uint32_t (&K)[EPL], uint32_t (&V)[EPL], uint32_t d, uint32_t nv, bool lane0) {
  uint32_t pk = __shfl_up_sync(FULL_MASK, K[EPL - 1], 1);
  const uint32_t pv = __shfl_up_sync(FULL_MASK, V[EPL - 1], 1);
  if (lane0) pk = 0u;  // nothing below position 0: "the entry below stays"
  // Slot e keeps its entry while key <= d (the new one lands after its equals); otherwise it takes the new
  // entry if the slot below keeps its own, else the entry of the slot below.  One predicated select per
  // register, highest slot first so that every source is still the old value.
#pragma unroll
  for (int e = EPL - 1; e >= 0; e--) {
    const uint32_t prk = e > 0 ? K[e - 1] : pk;
    const uint32_t prv = e > 0 ? V[e - 1] : pv;
    asm("{\n"
        ".reg .pred stay, here;\n"
        "setp.le.u32 stay, %0, %2;\n"
        "setp.le.u32 here, %3, %2;\n"
        "@!stay selp.u32 %0, %2, %3, here;\n"
        "@!stay selp.u32 %1, %4, %5, here;\n"
        "}\n"
        : "+r"(K[e]), "+r"(V[e])
        : "r"(d), "r"(prk), "r"(nv), "r"(prv));
  }
}

// nearest not-yet-expanded entry of one lane's slots, as a running (key, value) minimum: expanded and empty slots
// count as KEY_MAX (their flag bit smeared over the key); strict < keeps the lowest slot among equal keys
template <int EPL>
__device__ __forceinline__ void unexpanded_min(const uint32_t (&K)[EPL], const uint32_t (&V)[EPL], uint32_t &bk, uint32_t &bv) {
#pragma unroll
  for (int e = 0; e < EPL; e++) {
    const uint32_t c = K[e] | (uint32_t)((int32_t)V[e] >> 31);
    if (c < bk) {
      bk = c;
      bv = V[e];
    }
  }
}

template <int EPL>
__device__ __forceinline__ uint32_t list_key_at(const uint32_t (&K)[EPL], int lane_of, int slot_of) {
  uint32_t sel = K[0];
#pragma unroll
  for (int e = 1; e < EPL; e++)
    if (slot_of == e) sel = K[e];
  return __shfl_sync(FULL_MASK, sel, lane_of);
}

// sequential-j accumulation over one vector of coordinates; every sub / mul / add rounded on its own (no FMA)
__device__ __forceinline__ float acc_l2(float a, const float2 w, const float2 x) {
  float t = __fsub_rn(w.x, x.x);
  a = __fadd_rn(a, __fmul_rn(t, t));
  t = __fsub_rn(w.y, x.y);
  return __fadd_rn(a, __fmul_rn(t, t));
}
__device__ __forceinline__ float acc_l2(float a, const float4 w, const float4 x) {
  a = acc_l2(a, make_float2(w.x, w.y), make_float2(x.x, x.y));
  return acc_l2(a, make_float2(w.z, w.w), make_float2(x.z, x.w));
}
__device__ __forceinline__ float acc_ip(float a, const float2 w, const float2 x) {
  a = __fadd_rn(a, __fmul_rn(w.x, x.x));
  return __fadd_rn(a, __fmul_rn(w.y, x.y));
}
__device__ __forceinline__ float acc_ip(float a, const float4 w, const float4 x) {
  a = acc_ip(a, make_float2(w.x, w.y), make_float2(x.x, x.y));
  return acc_ip(a, make_float2(w.z, w.w), make_float2(x.z, x.w));
}

// ---- K1 inside the walk: build this query's table into T (shared) ----------------------------------
// cbt is the transposed codebook [m][j/V][c][V]; the query is staged in the tail rows of T itself (they are
// overwritten last, after their part of the query has been consumed; the host checks that this holds).
template <int M, int V>
__device__ __forceinline__ void build_table(float *T, const float *__restrict__ qg, const float *__restrict__ cbt, int ds,
                                            int is_ip, float bias, int lane) {
  typedef typename std::conditional<V == 4, float4, float2>::type vec_t;
  const int D = M * ds;
  const int R = (D + 255) >> 8;
  float *stage = T + (M - R) * 256;
  for (int i = lane; i < D; i += 32) stage[i] = __ldg(qg + i);
  __syncwarp();
  const int nv = ds / V;
  const vec_t *cb = reinterpret_cast<const vec_t *>(cbt);
  for (int m = 0; m < M; m++) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = 0.f;
    const vec_t *xq = reinterpret_cast<const vec_t *>(stage + m * ds);
    const vec_t *cm = cb + (size_t)m * nv * 256 + lane;
    if (!is_ip) {
      for (int jv = 0; jv < nv; jv++) {
        const vec_t x = xq[jv];
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = acc_l2(acc[i], __ldg(cm + jv * 256 + 32 * i), x);
      }
    } else {
      for (int jv = 0; jv < nv; jv++) {
        const vec_t x = xq[jv];
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = acc_ip(acc[i], __ldg(cm + jv * 256 + 32 * i), x);
      }
    }
    __syncwarp();  // every lane has read q_m (and all before it): row m may now overwrite staged floats
#pragma unroll
    for (int i = 0; i < 8; i++) T[m * 256 + lane + 32 * i] = is_ip ? __fsub_rn(bias, acc[i]) : acc[i];
  }
  __syncwarp();
}

// ---- greedy descent maxlevel..1 (hnswalg.h:1245-1274): after scanning one node's list the reference holds the
// FIRST minimum among the neighbours that beat curdist (strict <, sequential).  Out: the level-0 entry node and the
// order-preserving image of its distance; hops / nbrs / evals are advanced as the reference's counters are ----
template <int M>
__device__ __forceinline__ void descend4(const GraphDev &g, const float *T, const int lane, const bool has_slotu, int &hops, int &nbrs,
                                         int &evals, uint32_t &cur_uk, uint32_t &rec) {
  {
    float r = 0.f;
#pragma unroll
    for (int m = 0; m < M; m++) r = __fadd_rn(r, T[m * 256 + g.ep_code[m]]);  // dist to the entry point (:1246)
    cur_uk = f2u(r);
  }
  rec = g.ep_rec;
  for (int level = g.maxlevel; level > 0; level--) {
    const uint8_t *base = g.up + g.up_off[level];
    bool changed = true;
    while (changed) {
      changed = false;
      const uint8_t *r = base + (size_t)rec * g.recu_bytes;
      hops++;
      uint32_t link = EMPTY_LINK;
      uint32_t cw[M / 4];
#pragma unroll
      for (int i = 0; i < M / 4; i++) cw[i] = 0u;
      if (has_slotu) {
        link = __ldg(reinterpret_cast<const uint32_t *>(r) + lane);
        load_codes<M>(cw, r + g.code_offu + (size_t)lane * M);
      }
      const bool valid = link != EMPTY_LINK;
      const uint32_t uk = valid ? f2u(pq_score<M>(T, cw)) : KEY_MAX;
      const int nv = __popc(__ballot_sync(FULL_MASK, valid));
      nbrs += nv;
      evals += nv;
      const uint32_t mn = __reduce_min_sync(FULL_MASK, uk);
      if (mn < cur_uk) {
        const int src = __ffs(__ballot_sync(FULL_MASK, uk == mn)) - 1;  // first index wins ties
        rec = __shfl_sync(FULL_MASK, link, src);
        cur_uk = mn;
        changed = true;
      }
    }
    // step down: record index on the level below (node id when level == 1)
    rec = __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)rec * g.recu_bytes + g.tail_offu) + 1);
  }
}

// ---- launch geometry.  Shared memory per query = its table (M KB); the TMA form adds one 8-byte mbarrier per warp.
// An SM has 228 KB of shared memory and every resident CTA costs 1 KB on top of what it asks for, so at M=8
// 4 CTAs x 7 warps x 8 KB + 4 KB fills it to the byte: 28 queries per SM in CTAs small enough that the tail of one
// launch frees SMs piecewise for the next (the two lanes of annb_search_submit overlap that way).  The TMA form
// (8 bytes more per warp) runs 3 CTAs x 9 warps = 27.  Wider lists need more registers: fewer warps.  hnsw_walk4f
// (two lists of EP, EN <= 4 or 8 entries; ptxas: 64 registers at EP=2, EN=4, no spills) runs the EPL <= 4 shape.
constexpr int W4_SMEM_SM = 233472;  // 228 KB per SM
constexpr int w4_cta_warps(int M, int EPL, bool fused) {
  return M == 8 ? (EPL <= 4 ? (fused ? 7 : 9) : (EPL == 8 ? 5 : 7)) : 7;
}
constexpr int w4_ctas(int M, int EPL, bool fused) {
  return M == 8 ? (EPL <= 4 ? (fused ? 4 : 3) : (EPL == 8 ? 4 : 2)) : (M == 16 ? 2 : 1);
}
constexpr int w4_smem(int M, int EPL, bool fused) { return w4_cta_warps(M, EPL, fused) * (M * 1024 + (fused ? 0 : 8)); }
constexpr bool w4_fits(int M, int EPL, bool fused) {
  return w4_ctas(M, EPL, fused) * (w4_smem(M, EPL, fused) + 1024) <= W4_SMEM_SM;
}
constexpr int w4_max_threads(int M, int EPL) {
  return 32 * (w4_cta_warps(M, EPL, true) > w4_cta_warps(M, EPL, false) ? w4_cta_warps(M, EPL, true) : w4_cta_warps(M, EPL, false));
}
constexpr int w4_min_ctas(int M, int EPL) {  // register cap = 64K / (max threads x this): must allow either residency
  const int tf = w4_ctas(M, EPL, true) * w4_cta_warps(M, EPL, true) * 32, tt = w4_ctas(M, EPL, false) * w4_cta_warps(M, EPL, false) * 32;
  return (tf > tt ? tf : tt) / w4_max_threads(M, EPL);
}

// One launch of hnsw_walk4 / hnsw_walk4f in the EPL shape: kern(h->gd, p, args...).  The warps_per_cta / ctas_per_sm
// options cap the shape, and small batches are spread over all SMs instead of filling a few of them.
template <int M, int EPL, typename Kern, typename... Args>
int launch_w4(annb_index *h, Kern kern, const SearchParams &p_in, Args... args) {
  static_assert(w4_fits(M, EPL, true) && w4_fits(M, EPL, false), "walk4 geometry exceeds the SM's shared memory");
  SearchParams p = p_in;
  const bool fused = p.queries != nullptr;
  int warps = w4_cta_warps(M, EPL, fused), ctas = w4_ctas(M, EPL, fused);
  if (h->opt_warps_per_cta > 0) warps = (int)std::min<int64_t>(h->opt_warps_per_cta, warps);
  if (h->opt_ctas_per_sm > 0) ctas = (int)std::min<int64_t>(h->opt_ctas_per_sm, ctas);
  const int64_t per_sm = (p.B + h->sm_count - 1) / h->sm_count;
  if (per_sm < (int64_t)warps * ctas) {
    ctas = (int)std::max<int64_t>(1, std::min<int64_t>(ctas, (per_sm + warps - 1) / warps));
    if (ctas == 1) warps = (int)std::max<int64_t>(1, std::min<int64_t>(warps, per_sm));
  }
  const int smem = warps * (M * 1024 + (fused ? 0 : 8));
  ANNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 std::max(w4_smem(M, EPL, true), w4_smem(M, EPL, false))));
  ANNB_TRY_RC(walk_counter(h, p));
  const int blocks = (int)std::min<int64_t>((int64_t)h->sm_count * ctas, (p.B + warps - 1) / warps);
  kern<<<blocks, warps * 32, smem, h->stream>>>(h->gd, p, args...);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}


}  // namespace
