// adc_scan.cu -- K2: exhaustive ADC scan, plain (dist_pqcodes_to_codebooks) and fused with top-k
// (PQIndex.search), plus the (dist, id) k-way merge used for chunk partials and shard results.
//
// d[n] = sum_m T[m, code[n,m]], m sequential from 0.f     bindings/pq_bindings.pyx:30-47, :52-80
// top-k: k smallest ascending, ties by row index          pq_index.py:29-56 + annlite/math.py:94-120
//        (numpy leaves tie order unspecified; (dist, index) is the rule the oracle fixes too)
//
// Mapping (scan_topk): a CTA stages QT query tables in shared memory (one per warp) and streams a
// chunk of the code matrix; each lane scores one code row per step (coalesced code loads, L1
// shared by the CTA's warps), and the warp keeps its query's running top-k in a register-
// resident sorted list with a threshold test, so inserts are rare after warm-up.  Partials
// (B, chunks, k) are merged by merge_topk_kernel.  Bound: shared-memory gather rate for N*M
// small (C1: 80 KB of codes, L2/L1 resident), HBM reads of N*M bytes per query tile otherwise.
#include <math_constants.h>

#include "annb_internal.h"
#include "warp_list.cuh"

namespace {

template <typename code_t>
__device__ __forceinline__ float adc_lookup_row(const float *__restrict__ T, const code_t *__restrict__ row, int M,
                                                int Ks) {
  float r = 0.f;
  for (int m = 0; m < M; m++) r = __fadd_rn(r, T[m * Ks + (int)row[m]]);
  return r;
}

// specialisation for 8 one-byte codes (M = 8): one 64-bit load per row
__device__ __forceinline__ float adc_lookup_u8x8(const float *__restrict__ T, uint2 c, int Ks) {
  float r = 0.f;
  r = __fadd_rn(r, T[0 * Ks + (c.x & 0xff)]);
  r = __fadd_rn(r, T[1 * Ks + ((c.x >> 8) & 0xff)]);
  r = __fadd_rn(r, T[2 * Ks + ((c.x >> 16) & 0xff)]);
  r = __fadd_rn(r, T[3 * Ks + (c.x >> 24)]);
  r = __fadd_rn(r, T[4 * Ks + (c.y & 0xff)]);
  r = __fadd_rn(r, T[5 * Ks + ((c.y >> 8) & 0xff)]);
  r = __fadd_rn(r, T[6 * Ks + ((c.y >> 16) & 0xff)]);
  r = __fadd_rn(r, T[7 * Ks + (c.y >> 24)]);
  return r;
}

template <typename code_t>
__global__ void scan_kernel(const float *__restrict__ table, const code_t *__restrict__ codes, float *__restrict__ out,
                            int64_t N, int M, int Ks, int table_in_smem) {
  extern __shared__ float sT[];
  const float *T = table;
  if (table_in_smem) {
    for (int i = threadIdx.x; i < M * Ks; i += blockDim.x) sT[i] = table[i];
    __syncthreads();
    T = sT;
  }
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (int64_t)gridDim.x * blockDim.x) {
    float d;
    if (sizeof(code_t) == 1 && M == 8) {
      uint2 c = *reinterpret_cast<const uint2 *>(codes + n * 8);
      d = adc_lookup_u8x8(T, c, Ks);
    } else {
      d = adc_lookup_row<code_t>(T, codes + n * M, M, Ks);
    }
    out[n] = d;
  }
}

// partial top-k of one (query, chunk): results to part_d/part_i [(b*chunks + chunk)*k ...]
template <int EPL, typename code_t>
__global__ void __launch_bounds__(256)
scan_topk_kernel(const float *__restrict__ tables, const code_t *__restrict__ codes, int64_t B, int64_t N, int M, int Ks,
                 int k, int chunks, int64_t rows_per_chunk, int table_in_smem, float *__restrict__ part_d,
                 uint32_t *__restrict__ part_i) {
  extern __shared__ float sT[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int W = blockDim.x >> 5;
  const int64_t b = (int64_t)blockIdx.y * W + warp;
  const int chunk = blockIdx.x;
  const int TS = M * Ks;
  const float *T = nullptr;
  if (b < B) {
    T = tables + b * TS;
    if (table_in_smem) {
      float *dst = sT + warp * TS;
      for (int i = lane; i < TS; i += 32) dst[i] = T[i];
      T = dst;
    }
  }
  __syncwarp();
  if (b >= B) return;
  WarpList<EPL> L;
  L.clear();
  float worst = CUDART_INF_F;
  const int64_t r0 = (int64_t)chunk * rows_per_chunk;
  const int64_t r1 = min(N, r0 + rows_per_chunk);
  for (int64_t base = r0; base < r1; base += 32) {
    const int64_t n = base + lane;
    float d = CUDART_INF_F;
    if (n < r1) {
      if (sizeof(code_t) == 1 && M == 8) {
        uint2 c = *reinterpret_cast<const uint2 *>(codes + n * 8);
        d = adc_lookup_u8x8(T, c, Ks);
      } else {
        d = adc_lookup_row<code_t>(T, codes + n * M, M, Ks);
      }
    }
    unsigned mask = __ballot_sync(FULL_MASK, d < worst);
    while (mask) {
      const int j = __ffs(mask) - 1;
      mask &= mask - 1;
      const float dj = __shfl_sync(FULL_MASK, d, j);
      if (dj < worst) {
        L.insert(dj, (uint32_t)(base + j - r0), k);
        worst = L.key_at(k - 1);
      }
    }
  }
  // write the k best (positions 0..k-1), row index made global
#pragma unroll
  for (int e = 0; e < EPL; e++) {
    const int pos = e * 32 + lane;
    if (pos < k) {
      const int64_t o = (b * chunks + chunk) * k + pos;
      part_d[o] = L.k[e];
      part_i[o] = L.v[e] == LIST_EMPTY_VAL ? LIST_EMPTY_VAL : (uint32_t)(L.v[e] + r0);
    }
  }
}

// ---- query-tiled scan (round 2): lanes = QUERIES, not rows --------------------------------------------------
// scan_topk_kernel gives every warp its own table and lets its 32 lanes look up 32 DIFFERENT codes per step: 32
// random words of a 256-entry row land in the 32 banks ~3.5 deep, and the measured rate is 15 % of the shared-memory
// peak (bench.py k2_exhaustive_scan, 1M rows).  Here a CTA stages the tables of QT = 16 queries INTERLEAVED --
// sT[(m*Ks + c)*16 + q] -- and a half-warp scores ONE row for those 16 queries: its 16 lanes read 16 consecutive
// words (the code is the same for all of them), so a warp instruction touches two 64-byte runs: conflict-free or
// 2-way.  The row's 8 code bytes are loaded once per 16 queries.  Every lane keeps the running top-KK of ITS
// (query, row-parity) pair in registers (static indexing, bubble insertion -- rare once the threshold has settled);
// the two halves are merged by shuffles, and the per-warp lists (G = chunks x warps per query) go to
// merge_topk_kernel.  Same arithmetic (m sequential, fp32), same (dist, row) order: bit-identical results.
constexpr int QT = 16;
constexpr int TILED_WARPS = 16;

template <int KK>
__device__ __forceinline__ void lane_list_insert(float (&Kd)[KK], uint32_t (&Ki)[KK], float d, uint32_t id) {
  if (d < Kd[KK - 1] || (d == Kd[KK - 1] && id < Ki[KK - 1])) {
    Kd[KK - 1] = d;
    Ki[KK - 1] = id;
#pragma unroll
    for (int i = KK - 1; i > 0; i--) {
      const bool sw = Kd[i] < Kd[i - 1] || (Kd[i] == Kd[i - 1] && Ki[i] < Ki[i - 1]);
      const float td = Kd[i];
      const uint32_t ti = Ki[i];
      Kd[i] = sw ? Kd[i - 1] : td;
      Ki[i] = sw ? Ki[i - 1] : ti;
      Kd[i - 1] = sw ? td : Kd[i - 1];
      Ki[i - 1] = sw ? ti : Ki[i - 1];
    }
  }
}

template <int KK>
__global__ void __launch_bounds__(TILED_WARPS * 32, 1)
scan_topk_tiled_kernel(const float *__restrict__ tables, const uint8_t *__restrict__ codes, int64_t B, int64_t N, int Ks, int k,
                       int chunks, int64_t rows_per_chunk, float *__restrict__ part_d, uint32_t *__restrict__ part_i) {
  constexpr int M = 8;
  extern __shared__ float sT[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, q = lane & 15;
  const int64_t b0 = (int64_t)blockIdx.y * QT;
  const int chunk = blockIdx.x;
  const int TS = M * Ks;
  // stage the tile: thread -> (table entry i, query q), q fastest => conflict-free shared-memory stores
  for (int t = threadIdx.x; t < TS * QT; t += blockDim.x) {
    const int qq = t & (QT - 1), i = t >> 4;
    sT[t] = (b0 + qq < B) ? __ldg(tables + (b0 + qq) * TS + i) : 0.f;
  }
  __syncthreads();
  float Kd[KK];
  uint32_t Ki[KK];
#pragma unroll
  for (int i = 0; i < KK; i++) {
    Kd[i] = CUDART_INF_F;
    Ki[i] = LIST_EMPTY_VAL;
  }
  const int64_t r0 = (int64_t)chunk * rows_per_chunk;
  const int64_t r1 = min(N, r0 + rows_per_chunk);
  const float *Tq = sT + q;
  auto score = [&](const uint2 c) -> float {  // m sequential from 0.f, every add rounded (pq_bindings.pyx:30-47)
    float d = 0.f;
    d = __fadd_rn(d, Tq[(0 * Ks + (int)(c.x & 0xff)) * QT]);
    d = __fadd_rn(d, Tq[(1 * Ks + (int)((c.x >> 8) & 0xff)) * QT]);
    d = __fadd_rn(d, Tq[(2 * Ks + (int)((c.x >> 16) & 0xff)) * QT]);
    d = __fadd_rn(d, Tq[(3 * Ks + (int)(c.x >> 24)) * QT]);
    d = __fadd_rn(d, Tq[(4 * Ks + (int)(c.y & 0xff)) * QT]);
    d = __fadd_rn(d, Tq[(5 * Ks + (int)((c.y >> 8) & 0xff)) * QT]);
    d = __fadd_rn(d, Tq[(6 * Ks + (int)((c.y >> 16) & 0xff)) * QT]);
    d = __fadd_rn(d, Tq[(7 * Ks + (int)(c.y >> 24)) * QT]);
    return d;
  };
  // two rows per lane and iteration: two independent lookup chains in flight (16 warps per SM is all the tile leaves room for)
  constexpr int64_t STEP = 2 * TILED_WARPS;
  int64_t r = r0 + 2 * warp + half;
  for (; r + STEP < r1; r += 2 * STEP) {
    const uint2 ca = __ldg(reinterpret_cast<const uint2 *>(codes + r * 8));
    const uint2 cb = __ldg(reinterpret_cast<const uint2 *>(codes + (r + STEP) * 8));
    const float da = score(ca), db = score(cb);
    lane_list_insert<KK>(Kd, Ki, da, (uint32_t)r);
    lane_list_insert<KK>(Kd, Ki, db, (uint32_t)(r + STEP));
  }
  if (r < r1) {
    const uint2 ca = __ldg(reinterpret_cast<const uint2 *>(codes + r * 8));
    lane_list_insert<KK>(Kd, Ki, score(ca), (uint32_t)r);
  }
  // the odd-row half hands its list to the even-row half of the same query
#pragma unroll
  for (int i = 0; i < KK; i++) {
    const float od = __shfl_down_sync(FULL_MASK, Kd[i], 16);
    const uint32_t oi = __shfl_down_sync(FULL_MASK, Ki[i], 16);
    if (half == 0 && oi != LIST_EMPTY_VAL) lane_list_insert<KK>(Kd, Ki, od, oi);
  }
  if (half == 0 && b0 + q < B) {
    const int64_t G = (int64_t)chunks * TILED_WARPS;
    const int64_t o = ((b0 + q) * G + (int64_t)chunk * TILED_WARPS + warp) * k;
#pragma unroll
    for (int i = 0; i < KK; i++)
      if (i < k) {
        part_d[o + i] = Kd[i];
        part_i[o + i] = Ki[i];
      }
  }
}

// ---- the same, on a diet (ncu of the first version: 73 warp instructions per two-row step, 4.5 ms for 1000 queries x
// 1M rows, and 3 ms more in the merge of the 16 x chunks per-warp lists): Ks = 256 at compile time (lookup = byte
// extract + shift + LDS with an immediate row offset), the threshold test of the streaming loop compares distances only
// (rows arrive in ascending order, so an equal distance never displaces), and the CTA reduces its 16 per-warp lists
// to ONE list per (query, chunk) through shared memory before anything is written.
template <int KK>
__device__ __forceinline__ void lane_list_insert_ascending_rows(float (&Kd)[KK], uint32_t (&Ki)[KK], float d, uint32_t id) {
  if (d < Kd[KK - 1]) {
    Kd[KK - 1] = d;
    Ki[KK - 1] = id;
#pragma unroll
    for (int i = KK - 1; i > 0; i--) {
      const bool sw = Kd[i] < Kd[i - 1];
      const float td = Kd[i];
      const uint32_t ti = Ki[i];
      Kd[i] = sw ? Kd[i - 1] : td;
      Ki[i] = sw ? Ki[i - 1] : ti;
      Kd[i - 1] = sw ? td : Kd[i - 1];
      Ki[i - 1] = sw ? ti : Ki[i - 1];
    }
  }
}

template <int KK>
__global__ void __launch_bounds__(TILED_WARPS * 32, 1)
scan_topk_tiled2_kernel(const float *__restrict__ tables, const uint8_t *__restrict__ codes, int64_t B, int64_t N, int k, int chunks,
                        int64_t rows_per_chunk, float *__restrict__ part_d, uint32_t *__restrict__ part_i) {
  constexpr int M = 8, KS = 256;
  extern __shared__ float sT[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, q = lane & 15;
  const int64_t b0 = (int64_t)blockIdx.y * QT;
  const int chunk = blockIdx.x;
  constexpr int TS = M * KS;
  for (int t = threadIdx.x; t < TS * QT; t += blockDim.x) {
    const int qq = t & (QT - 1), i = t >> 4;
    sT[t] = (b0 + qq < B) ? __ldg(tables + (b0 + qq) * TS + i) : 0.f;
  }
  __syncthreads();
  float Kd[KK];
  uint32_t Ki[KK];
#pragma unroll
  for (int i = 0; i < KK; i++) {
    Kd[i] = CUDART_INF_F;
    Ki[i] = LIST_EMPTY_VAL;
  }
  const int64_t r0 = (int64_t)chunk * rows_per_chunk;
  const int64_t r1 = min(N, r0 + rows_per_chunk);
  const float *Tq = sT + q;
  auto score = [&](const uint2 c) -> float {  // m sequential from 0.f, every add rounded (pq_bindings.pyx:30-47)
    float d = 0.f;
    d = __fadd_rn(d, Tq[((c.x & 0xffu) + 0 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.x >> 8) & 0xffu) + 1 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.x >> 16) & 0xffu) + 2 * KS) * QT]);
    d = __fadd_rn(d, Tq[((c.x >> 24) + 3 * KS) * QT]);
    d = __fadd_rn(d, Tq[((c.y & 0xffu) + 4 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.y >> 8) & 0xffu) + 5 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.y >> 16) & 0xffu) + 6 * KS) * QT]);
    d = __fadd_rn(d, Tq[((c.y >> 24) + 7 * KS) * QT]);
    return d;
  };
  constexpr int64_t STEP = 2 * TILED_WARPS;
  int64_t r = r0 + 2 * warp + half;
  for (; r + STEP < r1; r += 2 * STEP) {
    const uint2 ca = __ldg(reinterpret_cast<const uint2 *>(codes + r * 8));
    const uint2 cb = __ldg(reinterpret_cast<const uint2 *>(codes + (r + STEP) * 8));
    const float da = score(ca), db = score(cb);
    lane_list_insert_ascending_rows<KK>(Kd, Ki, da, (uint32_t)r);
    lane_list_insert_ascending_rows<KK>(Kd, Ki, db, (uint32_t)(r + STEP));
  }
  if (r < r1) {
    const uint2 ca = __ldg(reinterpret_cast<const uint2 *>(codes + r * 8));
    lane_list_insert_ascending_rows<KK>(Kd, Ki, score(ca), (uint32_t)r);
  }
  // the odd-row half hands its list to the even-row half of the same query: (dist, row) order from here on
#pragma unroll
  for (int i = 0; i < KK; i++) {
    const float od = __shfl_down_sync(FULL_MASK, Kd[i], 16);
    const uint32_t oi = __shfl_down_sync(FULL_MASK, Ki[i], 16);
    if (half == 0 && oi != LIST_EMPTY_VAL) lane_list_insert<KK>(Kd, Ki, od, oi);
  }
  // ---- CTA reduction: the 16 per-warp lists of a query -> one list, through the (no longer needed) table area ----
  __syncthreads();  // every warp is done with the tables
  float *sd = sT;
  uint32_t *si = reinterpret_cast<uint32_t *>(sT + QT * TILED_WARPS * KK);
  if (half == 0) {
#pragma unroll
    for (int i = 0; i < KK; i++) {
      sd[(q * TILED_WARPS + warp) * KK + i] = Kd[i];
      si[(q * TILED_WARPS + warp) * KK + i] = Ki[i];
    }
  }
  __syncthreads();
  // warp w finishes query w: lane l < 16 holds the list warp l produced, the other lanes hold empty lists
#pragma unroll
  for (int i = 0; i < KK; i++) {
    Kd[i] = half == 0 ? sd[(warp * TILED_WARPS + q) * KK + i] : CUDART_INF_F;
    Ki[i] = half == 0 ? si[(warp * TILED_WARPS + q) * KK + i] : LIST_EMPTY_VAL;
  }
  const int64_t b = b0 + warp;
  const int64_t o = (b * chunks + chunk) * k;
  for (int j = 0; j < k; j++) {
    float md = Kd[0];
    uint32_t mi = Ki[0];
#pragma unroll
    for (int s2 = 16; s2 > 0; s2 >>= 1) {
      const float od = __shfl_xor_sync(FULL_MASK, md, s2);
      const uint32_t oi = __shfl_xor_sync(FULL_MASK, mi, s2);
      if (od < md || (od == md && oi < mi)) {
        md = od;
        mi = oi;
      }
    }
    if (lane == 0 && b < B) {
      part_d[o + j] = md;
      part_i[o + j] = mi;
    }
    if (Ki[0] == mi && mi != LIST_EMPTY_VAL) {  // row ids are unique across the lists: exactly one lane pops its head
#pragma unroll
      for (int i = 0; i + 1 < KK; i++) {
        Kd[i] = Kd[i + 1];
        Ki[i] = Ki[i + 1];
      }
      Kd[KK - 1] = CUDART_INF_F;
      Ki[KK - 1] = LIST_EMPTY_VAL;
    }
  }
}

// Merge G sorted (ascending) lists of k (dist, id) per query into the global k best, ordered
// by (dist, id).  One warp per query; lists are tiny (G*k entries).  Used for chunk partials
// (ids = u32 row index -> i64) and for shard results (ids = u64 labels).
// CellContainer.ivf_search merge: annlite/container.py:130-138 (hstack -> argsort[:limit]).
template <typename in_id_t, typename out_id_t, int EPL>
__global__ void merge_topk_kernel(const float *__restrict__ d_in, const in_id_t *__restrict__ i_in, int G, int64_t B, int k,
                                  int64_t g_stride, int64_t b_stride, float *__restrict__ d_out,
                                  out_id_t *__restrict__ i_out, in_id_t empty_in, out_id_t empty_out) {
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  // Rank-based merge: entry x gets rank = #{y : (d_y, id_y) < (d_x, id_x)}; ranks < k are written.
  // G*k is small (<= a few thousand), O((G*k)^2 / 32) per query is negligible next to the scan / walk.
  const int total = G * k;
  for (int x = lane; x < total; x += 32) {
    const int gx = x / k, px = x - gx * k;
    const float dx = d_in[gx * g_stride + b * b_stride + px];
    const in_id_t ix = i_in[gx * g_stride + b * b_stride + px];
    if (ix == empty_in) continue;
    int rank = 0;
    for (int y = 0; y < total; y++) {
      const int gy = y / k, py = y - gy * k;
      const float dy = d_in[gy * g_stride + b * b_stride + py];
      const in_id_t iy = i_in[gy * g_stride + b * b_stride + py];
      if (iy == empty_in) continue;
      rank += (dy < dx) || (dy == dx && (iy < ix || (iy == ix && y < x)));
    }
    if (rank < k) {
      d_out[b * k + rank] = dx;
      i_out[b * k + rank] = (out_id_t)ix;
    }
  }
  // fill the tail when fewer than k valid entries exist
  int valid = 0;
  for (int x = lane; x < total; x += 32) {
    const int gx = x / k, px = x - gx * k;
    valid += i_in[gx * g_stride + b * b_stride + px] != empty_in;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) valid += __shfl_xor_sync(FULL_MASK, valid, o);
  for (int p = valid + lane; p < k; p += 32) {
    d_out[b * k + p] = CUDART_INF_F;
    i_out[b * k + p] = empty_out;
  }
}

}  // namespace

static size_t smem_optin_limit(int device) {
  int v = 0;
  cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  return (size_t)v;
}

int launch_scan(annb_index *h, const float *d_table, float *d_out) {
  const int64_t N = h->n_codes;
  if (N == 0) return ANNB_OK;
  const size_t tbytes = (size_t)h->M * h->Ks * sizeof(float);
  const int in_smem = tbytes <= 96 * 1024;
  int blocks = (int)std::min<int64_t>((N + 255) / 256, (int64_t)h->sm_count * 8);
  if (h->code_bytes == 1) {
    if (in_smem && tbytes > 48 * 1024)
      ANNB_CUDA(cudaFuncSetAttribute(scan_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tbytes));
    scan_kernel<uint8_t><<<blocks, 256, in_smem ? tbytes : 0, h->stream>>>(d_table, (const uint8_t *)h->d_codes, d_out, N,
                                                                         h->M, h->Ks, in_smem);
  } else {
    if (in_smem && tbytes > 48 * 1024)
      ANNB_CUDA(cudaFuncSetAttribute(scan_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tbytes));
    scan_kernel<uint16_t><<<blocks, 256, in_smem ? tbytes : 0, h->stream>>>(d_table, (const uint16_t *)h->d_codes, d_out,
                                                                          N, h->M, h->Ks, in_smem);
  }
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

template <int EPL, typename code_t>
static int run_scan_topk(annb_index *h, const float *d_tables, int64_t B, int k, int chunks, int64_t rows_per_chunk,
                         int W, int in_smem, size_t smem, float *part_d, uint32_t *part_i) {
  auto kern = scan_topk_kernel<EPL, code_t>;
  if (smem > 48 * 1024) ANNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t done = 0;
  while (done < B) {
    int64_t nb = std::min<int64_t>(B - done, (int64_t)65535 * W);
    dim3 grid((unsigned)chunks, (unsigned)((nb + W - 1) / W));
    kern<<<grid, W * 32, smem, h->stream>>>(d_tables + done * h->M * h->Ks, (const code_t *)h->d_codes, nb, h->n_codes,
                                            h->M, h->Ks, k, chunks, rows_per_chunk, in_smem,
                                            part_d + done * chunks * k, part_i + done * chunks * k);
    h->launches++;
    ANNB_CUDA(cudaGetLastError());
    done += nb;
  }
  return ANNB_OK;
}

// the query-tiled scan: M = 8 one-byte codes, a 16-query interleaved tile that fits shared memory, k <= 16 (per-lane
// register lists), enough queries to fill tiles and enough rows to amortise staging a 128 KB tile
template <int KK>
static int run_scan_topk_tiled(annb_index *h, const float *d_tables, int64_t B, int k, int64_t *d_ids, float *d_dists) {
  const int64_t N = h->n_codes;
  const size_t smem = (size_t)h->M * h->Ks * QT * sizeof(float);
  const bool v2 = h->Ks == 256 && h->opt_scan_kernel != 3;   // the diet version: Ks = 256, one list per (query, chunk)
  auto kern = scan_topk_tiled_kernel<KK>;
  auto kern2 = scan_topk_tiled2_kernel<KK>;
  if (v2) ANNB_CUDA(cudaFuncSetAttribute(kern2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  else ANNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t tiles = (B + QT - 1) / QT;
  // one CTA per SM is resident (the tile): ~2 waves of CTAs, at most 16 chunks (the merge sees chunks x 16 lists)
  int chunks = (int)std::max<int64_t>(1, std::min<int64_t>(16, (2LL * h->sm_count + tiles - 1) / tiles));
  chunks = (int)std::min<int64_t>(chunks, std::max<int64_t>(1, N / 4096));
  int64_t rows_per_chunk = (N + chunks - 1) / chunks;
  rows_per_chunk = (rows_per_chunk + 31) / 32 * 32;
  chunks = (int)std::max<int64_t>(1, (N + rows_per_chunk - 1) / rows_per_chunk);
  const int G = v2 ? chunks : chunks * TILED_WARPS;
  float *part_d;
  uint32_t *part_i;
  int rc;
  if ((rc = annb_scratch(h, 16, (size_t)B * G * k * sizeof(float), (void **)&part_d))) return rc;
  if ((rc = annb_scratch(h, 17, (size_t)B * G * k * sizeof(uint32_t), (void **)&part_i))) return rc;
  int64_t done = 0;
  while (done < B) {
    const int64_t nb = std::min<int64_t>(B - done, (int64_t)65535 * QT);
    dim3 grid((unsigned)chunks, (unsigned)((nb + QT - 1) / QT));
    if (v2)
      kern2<<<grid, TILED_WARPS * 32, smem, h->stream>>>(d_tables + done * h->M * h->Ks, (const uint8_t *)h->d_codes, nb, N, k, chunks,
                                                         rows_per_chunk, part_d + done * G * k, part_i + done * G * k);
    else
      kern<<<grid, TILED_WARPS * 32, smem, h->stream>>>(d_tables + done * h->M * h->Ks, (const uint8_t *)h->d_codes, nb, N, h->Ks, k, chunks,
                                                        rows_per_chunk, part_d + done * G * k, part_i + done * G * k);
    h->launches++;
    ANNB_CUDA(cudaGetLastError());
    done += nb;
  }
  const int warps = 4;
  merge_topk_kernel<uint32_t, int64_t, 1><<<(unsigned)((B + warps - 1) / warps), warps * 32, 0, h->stream>>>(
      part_d, part_i, G, B, k, (int64_t)k, (int64_t)G * k, d_dists, d_ids, LIST_EMPTY_VAL, (int64_t)-1);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_scan_topk(annb_index *h, const float *d_tables, int64_t B, int k, int64_t *d_ids, float *d_dists) {
  if (B == 0) return ANNB_OK;
  const int64_t N = h->n_codes;
  if (k > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "k=%d exceeds the limit %d of the register-resident top-k list", k, ANNB_MAX_EF);
  if (N >= (int64_t)0xffffffffll) ANNB_FAIL(ANNB_ELIMIT, "scan supports < 2^32-1 rows per index (shard larger sets)");
  const size_t tbytes = (size_t)h->M * h->Ks * sizeof(float);
  const size_t lim = smem_optin_limit(h->device);
  if (h->opt_scan_kernel != 1 && h->M == 8 && h->code_bytes == 1 && k <= 16 && tbytes * QT + 1024 <= lim &&
      ((B >= 64 && N >= 32768) || h->opt_scan_kernel >= 2)) {
    if (k <= 1) return run_scan_topk_tiled<1>(h, d_tables, B, k, d_ids, d_dists);
    if (k <= 10) return run_scan_topk_tiled<10>(h, d_tables, B, k, d_ids, d_dists);
    return run_scan_topk_tiled<16>(h, d_tables, B, k, d_ids, d_dists);
  }
  int W = 8;
  int in_smem = 1;
  while (W > 1 && W * tbytes > lim - 1024) W >>= 1;
  if (W * tbytes > lim - 1024) in_smem = 0, W = 8;
  const size_t smem = in_smem ? W * tbytes : 0;
  // enough (tile, chunk) CTAs to fill the GPU for ~2 waves; chunks of >= 1024 rows
  const int64_t tiles = (B + W - 1) / W;
  int64_t want = std::max<int64_t>(1, (2LL * h->sm_count * 2 + tiles - 1) / tiles);
  int64_t maxchunks = std::max<int64_t>(1, N / 1024);
  int chunks = (int)std::min<int64_t>(std::min<int64_t>(want, maxchunks), 128);
  int64_t rows_per_chunk = (N + chunks - 1) / chunks;
  rows_per_chunk = (rows_per_chunk + 31) / 32 * 32;
  chunks = (int)std::max<int64_t>(1, (N + rows_per_chunk - 1) / rows_per_chunk);

  float *part_d;
  uint32_t *part_i;
  int rc;
  if ((rc = annb_scratch(h, 16, (size_t)B * chunks * k * sizeof(float), (void **)&part_d))) return rc;
  if ((rc = annb_scratch(h, 17, (size_t)B * chunks * k * sizeof(uint32_t), (void **)&part_i))) return rc;

  const int epl = (k + 31) / 32;
#define ST_CASE(E)                                                                                                    \
  if (h->code_bytes == 1)                                                                                             \
    rc = run_scan_topk<E, uint8_t>(h, d_tables, B, k, chunks, rows_per_chunk, W, in_smem, smem, part_d, part_i);      \
  else                                                                                                                \
    rc = run_scan_topk<E, uint16_t>(h, d_tables, B, k, chunks, rows_per_chunk, W, in_smem, smem, part_d, part_i);
  if (epl <= 1) {
    ST_CASE(1)
  } else if (epl <= 2) {
    ST_CASE(2)
  } else if (epl <= 4) {
    ST_CASE(4)
  } else if (epl <= 8) {
    ST_CASE(8)
  } else {
    ST_CASE(16)
  }
#undef ST_CASE
  if (rc) return rc;
  // merge chunk partials: lists laid out [b][chunk][k] => g_stride = k, b_stride = chunks*k
  const int warps = 4;
  merge_topk_kernel<uint32_t, int64_t, 1><<<(unsigned)((B + warps - 1) / warps), warps * 32, 0, h->stream>>>(
      part_d, part_i, chunks, B, k, (int64_t)k, (int64_t)chunks * k, d_dists, d_ids, LIST_EMPTY_VAL, (int64_t)-1);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

// Shard merge (container.py:130-138 with the (dist, label) order): G ascending lists of k per query, given as two
// strided arrays so that the all-gathered PACKED per-rank buffers ([B*k dists][B*k labels] per rank, one NCCL
// all-gather) are merged in place.  One warp per query: the G*k pairs are staged in shared memory, then every
// pair finds its global rank = its own position + sum over the other lists of a binary search (lists are sorted),
// O(G*k*G*log k / 32) per query instead of the all-pairs count.
__global__ void merge_sorted_kernel(const float *__restrict__ d_in, const uint64_t *__restrict__ l_in, int G, int64_t B, int k,
                                    int64_t d_gstride, int64_t l_gstride, float *__restrict__ d_out,
                                    uint64_t *__restrict__ l_out) {
  extern __shared__ __align__(16) unsigned char msm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int64_t b = (int64_t)blockIdx.x * nwarps + warp;
  if (b >= B) return;
  const int total = G * k;
  uint64_t *sl = reinterpret_cast<uint64_t *>(msm) + (size_t)warp * total;
  float *sd = reinterpret_cast<float *>(msm + (size_t)nwarps * total * 8) + (size_t)warp * total;
  for (int x = lane; x < total; x += 32) {
    const int g = x / k, p = x - g * k;
    sd[x] = d_in[g * d_gstride + b * k + p];
    sl[x] = l_in[g * l_gstride + b * k + p];
  }
  __syncwarp();
  int valid = 0;
  for (int x = lane; x < total; x += 32) {
    const uint64_t lx = sl[x];
    if (lx == UINT64_MAX) continue;  // a shard that found fewer than k
    valid++;
    const int gx = x / k;
    const float dx = sd[x];
    int rank = x - gx * k;  // pairs before it in its own (sorted) list
    for (int g = 0; g < G; g++) {
      if (g == gx) continue;
      // number of pairs of list g that precede (dx, lx): order (dist, label), equal pairs by list index
      int lo = 0, hi = k;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const float dm = sd[g * k + mid];
        const uint64_t lm = sl[g * k + mid];
        const bool before = lm != UINT64_MAX && (dm < dx || (dm == dx && (lm < lx || (lm == lx && g < gx))));
        if (before) lo = mid + 1;
        else hi = mid;
      }
      rank += lo;
    }
    if (rank < k) {
      d_out[b * k + rank] = dx;
      l_out[b * k + rank] = lx;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) valid += __shfl_xor_sync(FULL_MASK, valid, o);
  for (int p = valid + lane; p < k; p += 32) {
    d_out[b * k + p] = CUDART_INF_F;
    l_out[b * k + p] = UINT64_MAX;
  }
}

int launch_merge_topk(annb_index *h, const uint64_t *labels, const float *dists, int G, int64_t B, int k, int64_t l_gstride,
                      int64_t d_gstride, uint64_t *labels_out, float *dists_out, cudaStream_t stream) {
  if (B == 0) return ANNB_OK;
  const size_t per_warp = (size_t)G * k * 12;
  if (per_warp > 200 * 1024) ANNB_FAIL(ANNB_ELIMIT, "G*k=%d is too large for the shard merge", G * k);
  int warps = (int)std::max<size_t>(1, std::min<size_t>(8, (96 * 1024) / per_warp));
  const size_t smem = warps * per_warp;
  if (smem > 48 * 1024) ANNB_CUDA(cudaFuncSetAttribute(merge_sorted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  merge_sorted_kernel<<<(unsigned)((B + warps - 1) / warps), warps * 32, smem, stream>>>(dists, labels, G, B, k, d_gstride, l_gstride,
                                                                                       dists_out, labels_out);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

// ---- the multi-subset exact scan (annb_cellset_search* with bruteforce thresholds or ANNB_CELLS_EXACT) --------
// A job is one subset of one cell (a prepared filter's admitted rows, a label list's live entries, or the cell's live
// rows) and the query rows that scan it.  Gather: every job's subset is compacted (bitmap, in internal-id order, as
// annb_filter_labels lists it; the live rows through the deletion bitmap read inverted) or read (id list, in order,
// repeats kept), and its code rows and labels are copied once from the cell's own-code array into a contiguous scratch
// -- three launches for all jobs; a cell without deletions is scanned in place.  Scan: one launch for all jobs, a CTA
// per tile of one job's queries.  k <= 16: scan_topk_tiled2's mapping (16 interleaved tables, a half-warp scores one
// row for 16 queries, per-lane register lists, one CTA reduction); larger k: a warp per query with its table in shared
// memory and a WarpList, as scan_topk_kernel.  Unchunked, each CTA's lists are final and go straight to the pair's row
// of the by-cell scratch.  When the tiles are too few to fill the GPU (subset_scan_chunk_rows), each tile is split
// into row chunks, one CTA each; the last CTA of a tile to finish merges its chunks' lists in the same launch.
// Arithmetic and order are K2's: d = sum_m T[m, code[m]] from 0.f in fp32, the k best by (distance, position in the
// subset) -- annb_scan_subset's bits and order, chunked or not.
namespace {

constexpr int GATHER_THREADS = 256;  // one bitmap word (or one list entry) per thread
constexpr int SCAN_WARP_TILE = 8;    // queries per CTA of the warp-per-query form
constexpr int SUBSET_MAX_CHUNKS = 16;       // a tile's chunk lists are merged by one lane each
constexpr int64_t SUBSET_MIN_CHUNK = 4096;  // rows: a chunk amortises staging its CTA's tables (128 KB for 16 queries)

// word w of a job's bitmap as it admits rows: a filter's as it is, the deletions (SUBSET_LIVE) inverted over the cell's rows
__device__ __forceinline__ uint32_t subset_word(const SubsetScan &J, int64_t w) {
  const uint32_t x = J.bits[w];
  if (J.kind != SUBSET_LIVE) return x;
  const int64_t valid = J.n_rows - w * 32;
  return ~x & (valid >= 32 ? 0xffffffffu : ((1u << valid) - 1u));
}

// pass 1: admitted rows per block of a job's bitmap
__global__ void __launch_bounds__(GATHER_THREADS) subset_count_kernel(const SubsetScan *__restrict__ jobs) {
  const SubsetScan &J = jobs[blockIdx.y];
  if (!J.bits) return;
  const int64_t nb = (J.nwords + GATHER_THREADS - 1) / GATHER_THREADS;
  if (blockIdx.x >= nb) return;
  __shared__ unsigned int s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  const int64_t w = (int64_t)blockIdx.x * GATHER_THREADS + threadIdx.x;
  unsigned int c = w < J.nwords ? __popc(subset_word(J, w)) : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s, c);
  __syncthreads();
  if (threadIdx.x == 0) J.block_offs[blockIdx.x] = s;
}

// pass 2: the block counts of each job's bitmap -> exclusive offsets (one thread per job: a few hundred blocks at most)
__global__ void subset_offsets_kernel(const SubsetScan *__restrict__ jobs, int J) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= J || !jobs[j].bits) return;
  const int64_t nb = (jobs[j].nwords + GATHER_THREADS - 1) / GATHER_THREADS;
  unsigned int *o = jobs[j].block_offs;
  unsigned int run = 0;
  for (int64_t b = 0; b < nb; b++) {
    const unsigned int c = o[b];
    o[b] = run;
    run += c;
  }
}

// pass 3: each admitted row (bitmap, in id order) or list entry -> its code row and label at its subset position
__global__ void __launch_bounds__(GATHER_THREADS) subset_gather_kernel(const SubsetScan *__restrict__ jobs) {
  const SubsetScan &J = jobs[blockIdx.y];
  const int64_t t = (int64_t)blockIdx.x * GATHER_THREADS + threadIdx.x;
  if (!J.bits) {
    if (!J.ids || blockIdx.x * (int64_t)GATHER_THREADS >= J.n) return;  // (a live-rows job without deletions: in place)
    if (t < J.n) {
      const uint32_t id = J.ids[t];
      reinterpret_cast<uint2 *>(J.codes)[t] = __ldg(reinterpret_cast<const uint2 *>(J.cell_codes) + id);
      J.labels[t] = J.cell_labels[id];
    }
    return;
  }
  if (blockIdx.x * (int64_t)GATHER_THREADS >= J.nwords) return;
  __shared__ unsigned int warp_sums[GATHER_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t word = t < J.nwords ? subset_word(J, t) : 0u;
  const unsigned int c = __popc(word);
  unsigned int x = c;  // inclusive scan over the warp, then over the warps
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int y = __shfl_up_sync(FULL_MASK, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  unsigned int before = 0;
  for (int w = 0; w < wid; w++) before += warp_sums[w];
  int64_t pos = (int64_t)J.block_offs[blockIdx.x] + before + x - c;
  while (word) {
    const int b = __ffs(word) - 1;
    word &= word - 1;
    const int64_t id = t * 32 + b;
    reinterpret_cast<uint2 *>(J.codes)[pos] = __ldg(reinterpret_cast<const uint2 *>(J.cell_codes) + id);
    J.labels[pos] = J.cell_labels[id];
    pos++;
  }
}

// the k best of a pair -> its row of the by-cell scratch, found = k, counters {0 hops, 0 neighbours, n rows scored}
__device__ __forceinline__ void subset_write_tail(const SubsetScan &J, int64_t row, int32_t *__restrict__ sfound,
                                                  int64_t *__restrict__ sstats) {
  sfound[row] = J.k;
  if (sstats) {
    sstats[row * 3 + 0] = 0;
    sstats[row * 3 + 1] = 0;
    sstats[row * 3 + 2] = J.n;
  }
}

// this CTA's chunk lists are written: true in the tile's last CTA to finish (which then reads every chunk's lists)
__device__ __forceinline__ bool subset_last_chunk(const SubsetScan &J, const SubsetChunks &ch, int group) {
  __shared__ int last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int nch = (unsigned int)((J.n + ch.rows - 1) / ch.rows);
    last = atomicAdd(ch.done + group, 1u) == nch - 1;
  }
  __syncthreads();
  if (last) __threadfence();
  return last;
}

// a query's chunk lists (list0 = its first; one per chunk of the subset, each K sorted (distance, position) entries)
// merged by one warp into the pair's row: lane l walks list l, and each step takes the smallest head by (distance,
// position) -- the unchunked scan's k best exactly
__device__ __forceinline__ void subset_merge_chunks(const SubsetScan &J, const SubsetChunks &ch, int64_t list0, int64_t row, int limit,
                                    uint64_t *__restrict__ sl, float *__restrict__ sd, int32_t *__restrict__ sfound,
                                    int64_t *__restrict__ sstats) {
  const int lane = threadIdx.x & 31;
  const int nch = (int)((J.n + ch.rows - 1) / ch.rows);
  const int64_t base = (list0 + lane) * ch.K;
  int h = 0;
  float d = CUDART_INF_F;
  uint32_t id = LIST_EMPTY_VAL;
  if (lane < nch) {
    d = __ldcg(ch.part_d + base);
    id = __ldcg(ch.part_i + base);
  }
  for (int j = 0; j < J.k; j++) {
    float md = d;
    uint32_t mi = id;
#pragma unroll
    for (int s2 = 16; s2 > 0; s2 >>= 1) {
      const float od = __shfl_xor_sync(FULL_MASK, md, s2);
      const uint32_t oi = __shfl_xor_sync(FULL_MASK, mi, s2);
      if (od < md || (od == md && oi < mi)) {
        md = od;
        mi = oi;
      }
    }
    if (lane == 0) {
      sd[row * limit + j] = md;
      sl[row * limit + j] = mi == LIST_EMPTY_VAL ? UINT64_MAX : J.labels[mi];
    }
    if (id == mi && mi != LIST_EMPTY_VAL) {  // positions are unique across the chunks: exactly one lane advances
      if (++h < ch.K) {
        d = __ldcg(ch.part_d + base + h);
        id = __ldcg(ch.part_i + base + h);
      } else {
        d = CUDART_INF_F;
        id = LIST_EMPTY_VAL;
      }
    }
  }
  if (lane == 0) subset_write_tail(J, row, sfound, sstats);
}

// tile i = (job, first query of the job); 16 queries per CTA, 16 warps
template <int KK>
__global__ void __launch_bounds__(TILED_WARPS * 32, 1)
subset_scan_tiled_kernel(const float *__restrict__ tables, const SubsetScan *__restrict__ jobs, const int4 *__restrict__ tiles,
                         const SubsetChunks ch, int n_cells, int limit, uint64_t *__restrict__ sl, float *__restrict__ sd,
                         int32_t *__restrict__ sfound, int64_t *__restrict__ sstats) {
  constexpr int M = 8, KS = 256, TS = M * KS;
  extern __shared__ float sT[];
  __shared__ int64_t srow[QT];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, q = lane & 15;
  const int4 tile = tiles[blockIdx.x];
  const SubsetScan &J = jobs[tile.x];
  const int q0 = tile.y, nq = min(QT, J.nq - q0);
  const bool chunked = ch.rows > 0;
  if (threadIdx.x < QT) srow[threadIdx.x] = threadIdx.x < nq ? (int64_t)J.queries[q0 + threadIdx.x] : -1;
  __syncthreads();
  for (int t = threadIdx.x; t < TS * QT; t += blockDim.x) {
    const int qq = t & (QT - 1), i = t >> 4;
    sT[t] = srow[qq] >= 0 ? __ldg(tables + srow[qq] * TS + i) : 0.f;
  }
  __syncthreads();
  float Kd[KK];
  uint32_t Ki[KK];
#pragma unroll
  for (int i = 0; i < KK; i++) {
    Kd[i] = CUDART_INF_F;
    Ki[i] = LIST_EMPTY_VAL;
  }
  const int64_t r0 = chunked ? (int64_t)tile.z * ch.rows : 0;
  const int64_t n = chunked ? min(J.n, r0 + ch.rows) : J.n;  // rows [r0, n) of the subset
  const uint8_t *codes = J.codes;
  const float *Tq = sT + q;
  auto score = [&](const uint2 c) -> float {  // m sequential from 0.f, every add rounded (pq_bindings.pyx:30-47)
    float d = 0.f;
    d = __fadd_rn(d, Tq[((c.x & 0xffu) + 0 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.x >> 8) & 0xffu) + 1 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.x >> 16) & 0xffu) + 2 * KS) * QT]);
    d = __fadd_rn(d, Tq[((c.x >> 24) + 3 * KS) * QT]);
    d = __fadd_rn(d, Tq[((c.y & 0xffu) + 4 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.y >> 8) & 0xffu) + 5 * KS) * QT]);
    d = __fadd_rn(d, Tq[(((c.y >> 16) & 0xffu) + 6 * KS) * QT]);
    d = __fadd_rn(d, Tq[((c.y >> 24) + 7 * KS) * QT]);
    return d;
  };
  constexpr int64_t STEP = 2 * TILED_WARPS;
  int64_t r = r0 + 2 * warp + half;
  for (; r + STEP < n; r += 2 * STEP) {
    const uint2 ca = __ldg(reinterpret_cast<const uint2 *>(codes + r * 8));
    const uint2 cb = __ldg(reinterpret_cast<const uint2 *>(codes + (r + STEP) * 8));
    const float da = score(ca), db = score(cb);
    lane_list_insert_ascending_rows<KK>(Kd, Ki, da, (uint32_t)r);
    lane_list_insert_ascending_rows<KK>(Kd, Ki, db, (uint32_t)(r + STEP));
  }
  if (r < n) {
    const uint2 ca = __ldg(reinterpret_cast<const uint2 *>(codes + r * 8));
    lane_list_insert_ascending_rows<KK>(Kd, Ki, score(ca), (uint32_t)r);
  }
  // the odd-row half hands its list to the even-row half of the same query: (dist, position) order from here on
#pragma unroll
  for (int i = 0; i < KK; i++) {
    const float od = __shfl_down_sync(FULL_MASK, Kd[i], 16);
    const uint32_t oi = __shfl_down_sync(FULL_MASK, Ki[i], 16);
    if (half == 0 && oi != LIST_EMPTY_VAL) lane_list_insert<KK>(Kd, Ki, od, oi);
  }
  // the 16 per-warp lists of a query -> one list, through the table area
  __syncthreads();
  float *rd = sT;
  uint32_t *ri = reinterpret_cast<uint32_t *>(sT + QT * TILED_WARPS * KK);
  if (half == 0) {
#pragma unroll
    for (int i = 0; i < KK; i++) {
      rd[(q * TILED_WARPS + warp) * KK + i] = Kd[i];
      ri[(q * TILED_WARPS + warp) * KK + i] = Ki[i];
    }
  }
  __syncthreads();
  // warp w finishes query w of the tile: lane l < 16 holds the list warp l produced
#pragma unroll
  for (int i = 0; i < KK; i++) {
    Kd[i] = half == 0 ? rd[(warp * TILED_WARPS + q) * KK + i] : CUDART_INF_F;
    Ki[i] = half == 0 ? ri[(warp * TILED_WARPS + q) * KK + i] : LIST_EMPTY_VAL;
  }
  // warp w < nq: the k best of query w's list -> its pair's row, or (chunked) the K best -> its chunk list
  const int64_t row = srow[warp] * n_cells + J.cell;
  const int64_t list0 = ((int64_t)tile.w * QT + warp) * ch.G;
  const int k = warp >= nq ? 0 : (chunked ? ch.K : J.k);
  for (int j = 0; j < k; j++) {
    float md = Kd[0];
    uint32_t mi = Ki[0];
#pragma unroll
    for (int s2 = 16; s2 > 0; s2 >>= 1) {
      const float od = __shfl_xor_sync(FULL_MASK, md, s2);
      const uint32_t oi = __shfl_xor_sync(FULL_MASK, mi, s2);
      if (od < md || (od == md && oi < mi)) {
        md = od;
        mi = oi;
      }
    }
    if (lane == 0 && chunked) {
      ch.part_d[(list0 + tile.z) * ch.K + j] = md;
      ch.part_i[(list0 + tile.z) * ch.K + j] = mi;
    } else if (lane == 0) {
      sd[row * limit + j] = md;
      sl[row * limit + j] = mi == LIST_EMPTY_VAL ? UINT64_MAX : J.labels[mi];
    }
    if (Ki[0] == mi && mi != LIST_EMPTY_VAL) {  // positions are unique across the lists: exactly one lane pops its head
#pragma unroll
      for (int i = 0; i + 1 < KK; i++) {
        Kd[i] = Kd[i + 1];
        Ki[i] = Ki[i + 1];
      }
      Kd[KK - 1] = CUDART_INF_F;
      Ki[KK - 1] = LIST_EMPTY_VAL;
    }
  }
  if (!chunked) {
    if (lane == 0 && warp < nq) subset_write_tail(J, row, sfound, sstats);
    return;
  }
  if (subset_last_chunk(J, ch, tile.w) && warp < nq) subset_merge_chunks(J, ch, list0, row, limit, sl, sd, sfound, sstats);
}

// k > 16: a warp per query (SCAN_WARP_TILE queries of one job per CTA), its table in shared memory, lanes over rows
template <int EPL>
__global__ void __launch_bounds__(SCAN_WARP_TILE * 32)
subset_scan_warp_kernel(const float *__restrict__ tables, const SubsetScan *__restrict__ jobs, const int4 *__restrict__ tiles,
                        const SubsetChunks ch, int n_cells, int limit, uint64_t *__restrict__ sl, float *__restrict__ sd,
                        int32_t *__restrict__ sfound, int64_t *__restrict__ sstats) {
  constexpr int TS = 8 * 256;
  extern __shared__ float sT[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int4 tile = tiles[blockIdx.x];
  const SubsetScan &J = jobs[tile.x];
  const int qi = tile.y + warp;
  const bool chunked = ch.rows > 0;
  if (qi >= J.nq && !chunked) return;  // (chunked: every warp takes part in the CTA's hand-over)
  const bool active = qi < J.nq;
  const int64_t qrow = active ? J.queries[qi] : 0;
  float *T = sT + warp * TS;
  for (int i = lane; i < TS; i += 32) T[i] = __ldg(tables + qrow * TS + i);
  __syncwarp();
  const int k = chunked ? ch.K : J.k;
  const int64_t r0 = chunked ? (int64_t)tile.z * ch.rows : 0;
  const int64_t n = !active ? 0 : (chunked ? min(J.n, r0 + ch.rows) : J.n);  // rows [r0, n) of the subset
  WarpList<EPL> L;
  L.clear();
  float worst = CUDART_INF_F;
  for (int64_t base = r0; base < n; base += 32) {
    const int64_t r = base + lane;
    float d = CUDART_INF_F;
    if (r < n) d = adc_lookup_u8x8(T, __ldg(reinterpret_cast<const uint2 *>(J.codes) + r), 256);
    unsigned mask = __ballot_sync(FULL_MASK, d < worst);
    while (mask) {
      const int j = __ffs(mask) - 1;
      mask &= mask - 1;
      const float dj = __shfl_sync(FULL_MASK, d, j);
      if (dj < worst) {
        L.insert(dj, (uint32_t)(base + j), k);
        worst = L.key_at(k - 1);
      }
    }
  }
  const int64_t row = qrow * n_cells + J.cell;
  if (!chunked) {
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const int pos = e * 32 + lane;
      if (pos < k) {
        sd[row * limit + pos] = L.k[e];
        sl[row * limit + pos] = L.v[e] == LIST_EMPTY_VAL ? UINT64_MAX : J.labels[L.v[e]];
      }
    }
    if (lane == 0) subset_write_tail(J, row, sfound, sstats);
    return;
  }
  const int64_t list0 = ((int64_t)tile.w * SCAN_WARP_TILE + warp) * ch.G;
  if (active) {
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const int pos = e * 32 + lane;
      if (pos < k) {
        ch.part_d[(list0 + tile.z) * ch.K + pos] = L.k[e];
        ch.part_i[(list0 + tile.z) * ch.K + pos] = L.v[e];
      }
    }
  }
  if (subset_last_chunk(J, ch, tile.w) && active) subset_merge_chunks(J, ch, list0, row, limit, sl, sd, sfound, sstats);
}

}  // namespace

bool subset_scan_applicable(const annb_index *h) { return h->M == 8 && h->code_bytes == 1 && h->Ks == 256; }

int subset_scan_tile_width(int kmax) { return kmax <= 16 ? QT : SCAN_WARP_TILE; }

// Unchunked while the tiles alone make two waves of CTAs (the tiled form holds one CTA per SM): every CTA's lists are
// then final, with no hand-over.  Fewer tiles -- a small batch over large subsets, such as whole cells -- are cut into
// chunks of at least SUBSET_MIN_CHUNK rows, at most SUBSET_MAX_CHUNKS per subset, enough for about two waves.
int64_t subset_scan_chunk_rows(const annb_index *h, int64_t tiles, int64_t longest) {
  const int64_t floor_rows = (longest + SUBSET_MAX_CHUNKS - 1) / SUBSET_MAX_CHUNKS;
  int64_t rows;
  if (h->opt_subset_chunk_rows != 0) {
    if (h->opt_subset_chunk_rows < 0) return 0;
    rows = std::max(h->opt_subset_chunk_rows, floor_rows);
  } else {
    const int64_t target = 2LL * h->sm_count;
    if (tiles <= 0 || tiles >= target) return 0;
    const int64_t g = std::min<int64_t>(SUBSET_MAX_CHUNKS, (target + tiles - 1) / tiles);
    rows = std::max<int64_t>(SUBSET_MIN_CHUNK, (longest + g - 1) / g);
    rows = (rows + 31) / 32 * 32;
  }
  return longest > rows ? rows : 0;
}

int launch_subset_scan(annb_index *h, cudaStream_t st, const SubsetScan *d_jobs, const std::vector<SubsetScan> &jobs,
                       const int4 *d_tiles, int64_t n_tiles, const SubsetChunks &ch, const float *tables, int n_cells, int limit,
                       uint64_t *sl, float *sd, int32_t *sfound, int64_t *sstats) {
  const int J = (int)jobs.size();
  if (J == 0 || n_tiles == 0) return ANNB_OK;
  if (J > 65535) ANNB_FAIL(ANNB_ELIMIT, "%d subsets in one scan (limit 65535)", J);
  int64_t gx = 1;
  int kmax = 1;
  bool any_bits = false;
  bool any_gather = false;
  for (const SubsetScan &s : jobs) {
    gx = std::max(gx, s.bits ? (s.nwords + GATHER_THREADS - 1) / GATHER_THREADS : (s.n + GATHER_THREADS - 1) / GATHER_THREADS);
    kmax = std::max(kmax, (int)s.k);
    any_bits |= s.bits != nullptr;
    any_gather |= s.bits != nullptr || s.ids != nullptr;
  }
  if (kmax > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "k=%d exceeds ANNB_MAX_EF=%d", kmax, ANNB_MAX_EF);
  if (ch.rows > 0 && (ch.K < kmax || ch.G > SUBSET_MAX_CHUNKS))
    ANNB_FAIL(ANNB_ESTATE, "internal: chunk lists of %d entries / %d chunks for k=%d", ch.K, ch.G, kmax);
  const dim3 ggrid((unsigned)gx, (unsigned)J);
  if (any_bits) {
    subset_count_kernel<<<ggrid, GATHER_THREADS, 0, st>>>(d_jobs);
    subset_offsets_kernel<<<(J + 127) / 128, 128, 0, st>>>(d_jobs, J);
    h->launches += 2;
  }
  if (any_gather) {
    subset_gather_kernel<<<ggrid, GATHER_THREADS, 0, st>>>(d_jobs);
    h->launches++;
    ANNB_CUDA(cudaGetLastError());
  }
  if (kmax <= 16) {
    const size_t smem = (size_t)8 * 256 * QT * sizeof(float);
#define SS_TILED(KKV)                                                                                                    \
  {                                                                                                                      \
    ANNB_CUDA(cudaFuncSetAttribute(subset_scan_tiled_kernel<KKV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    subset_scan_tiled_kernel<KKV><<<(unsigned)n_tiles, TILED_WARPS * 32, smem, st>>>(tables, d_jobs, d_tiles, ch, n_cells, limit, sl, \
                                                                                   sd, sfound, sstats);                \
  }
    if (kmax <= 1) SS_TILED(1)
    else if (kmax <= 10) SS_TILED(10)
    else SS_TILED(16)
#undef SS_TILED
  } else {
    const size_t smem = (size_t)SCAN_WARP_TILE * 8 * 256 * sizeof(float);
#define SS_WARP(E)                                                                                                       \
  {                                                                                                                      \
    ANNB_CUDA(cudaFuncSetAttribute(subset_scan_warp_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    subset_scan_warp_kernel<E><<<(unsigned)n_tiles, SCAN_WARP_TILE * 32, smem, st>>>(tables, d_jobs, d_tiles, ch, n_cells, limit, sl, \
                                                                                   sd, sfound, sstats);                \
  }
    const int epl = (kmax + 31) / 32;
    if (epl <= 1) SS_WARP(1)
    else if (epl <= 2) SS_WARP(2)
    else if (epl <= 4) SS_WARP(4)
    else if (epl <= 8) SS_WARP(8)
    else SS_WARP(16)
#undef SS_WARP
  }
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}
