// adc_table.cu -- K1: per-query ADC lookup tables, plus l2_normalize and PQ encode.
//
// Reference semantics (bit-exact):
//   L2 : T[b,m,c] = sum_j (cb[m,c,j] - q[b,m*ds+j])^2          bindings/pq_bindings.pyx:149-210
//   IP : T[b,m,c] = fp32(1/Ks) - sum_j cb[m,c,j]*q[b,m*ds+j]   pq_bindings.pyx:214-274 + pq.py:316-322
// j runs sequentially and every sub / mul / add is rounded separately (the reference is built
// in ISO C++ mode => no FMA contraction, SURVEY.md section 0.3), hence the explicit _rn
// intrinsics: nvcc's default -fmad=true would fuse and differ in the last ulp.
//
// Mapping: one thread = one codeword c of one subspace m; it keeps the ds codeword
// coordinates in registers and walks a tile of QT queries staged in shared memory, so the
// codebook (D*Ks*4 bytes, L2 resident) is read once per CTA and the (B,M,Ks) output is
// written as 1 KB coalesced rows.  The kernel is bound by that output write (HBM).
#include <math_constants.h>

#include "annb_internal.h"

namespace {

constexpr int K1_THREADS = 256;
constexpr int K1_QT = 32;  // queries per CTA

// DS > 0: compile-time subvector length, codeword in registers.  DS == 0: runtime ds; with `staged` the query tile and
// the CTA's codewords are copied to shared memory first, without it (ds too large for them to fit) both are read from
// global memory, where the codebook is L2 resident.  The arithmetic is the same either way.
template <int DS>
__global__ void __launch_bounds__(K1_THREADS)
adc_table_kernel(const float *__restrict__ q, const float *__restrict__ cb, float *__restrict__ out,
                 int64_t B, int M, int Ks, int ds_rt, int is_ip, float bias, int staged) {
  extern __shared__ float sm[];  // [K1_QT][ds] query sub-vectors, then (DS==0) [K1_THREADS][ds+1] codewords
  const int ds = DS > 0 ? DS : ds_rt;
  const int D = M * ds;
  const int chunks = (Ks + K1_THREADS - 1) / K1_THREADS;
  const int m = blockIdx.x / chunks;
  const int c = (blockIdx.x % chunks) * K1_THREADS + threadIdx.x;
  const int64_t b0 = (int64_t)blockIdx.y * K1_QT;
  const int nq = (int)min((int64_t)K1_QT, B - b0);

  const bool smem = DS > 0 || staged;
  const float *qs = smem ? sm : q + b0 * D + (int64_t)m * ds;
  const int qstride = smem ? ds : D;
  if (smem)
    for (int i = threadIdx.x; i < nq * ds; i += K1_THREADS) {
      int qi = i / ds, j = i - qi * ds;
      sm[i] = q[(b0 + qi) * D + (int64_t)m * ds + j];
    }
  float cw[DS > 0 ? DS : 1];
  const float *cws = sm + K1_QT * ds + threadIdx.x * (ds + 1);
  if (c < Ks) {
    const float *w = cb + ((size_t)m * Ks + c) * ds;
    if (DS > 0) {
#pragma unroll
      for (int j = 0; j < DS; j++) cw[j] = w[j];
    } else if (staged) {
      for (int j = 0; j < ds; j++) sm[K1_QT * ds + threadIdx.x * (ds + 1) + j] = w[j];
    } else {
      cws = w;
    }
  }
  if (smem) __syncthreads();
  if (c >= Ks) return;
  for (int qi = 0; qi < nq; qi++) {
    const float *x = qs + qi * qstride;
    float acc = 0.f;
    if (DS > 0) {
#pragma unroll
      for (int j = 0; j < DS; j++) {
        if (is_ip) {
          acc = __fadd_rn(acc, __fmul_rn(cw[j], x[j]));
        } else {
          float t = __fsub_rn(cw[j], x[j]);
          acc = __fadd_rn(acc, __fmul_rn(t, t));
        }
      }
    } else {
      for (int j = 0; j < ds; j++) {
        if (is_ip) {
          acc = __fadd_rn(acc, __fmul_rn(cws[j], x[j]));
        } else {
          float t = __fsub_rn(cws[j], x[j]);
          acc = __fadd_rn(acc, __fmul_rn(t, t));
        }
      }
    }
    if (is_ip) acc = __fsub_rn(bias, acc);
    out[((b0 + qi) * M + m) * (int64_t)Ks + c] = acc;
  }
}

// annlite/math.py:6-18: x / max(||x||, 1 if ||x|| < 10*eps).  One warp per row.  The sum order
// differs from numpy's einsum (SIMD, machine dependent), so this step is tolerance-level
// (<= 1 ulp on the norm), never bit-level -- see DESIGN.md "cosine".
__global__ void l2_normalize_kernel(float *__restrict__ x, int64_t B, int D) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B) return;
  float *r = x + row * D;
  float s = 0.f;
  for (int j = lane; j < D; j += 32) s = __fadd_rn(s, __fmul_rn(r[j], r[j]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  float nrm = __fsqrt_rn(s);
  if (nrm < 10.f * 1.1920929e-07f) nrm = 1.0f;
  for (int j = lane; j < D; j += 32) r[j] = __fdiv_rn(r[j], nrm);
}

// PQCodec.encode (annlite/core/codec/pq.py:158-177): nearest codeword per subspace, first minimum.  One warp per
// (row, subspace); lanes stride over codewords, fp32 squared distance with sequential j.  The reference delegates to
// scipy.cluster.vq.vq, whose rounding is BLAS dependent, so the chosen codeword is checked against a float64 argmin
// with a rounding bound (tests/numeric_bounds.py), not bit for bit.
// One order, `precedes`, serves the lane loop and the shuffle reduction: NaN counts as +inf and equal values go to
// the lower index.  A lane starts neutral (+inf, no index) and takes its first codeword whatever its distance, so
// the code is always < Ks and a row whose every distance overflows to +inf encodes to 0.  scipy refuses non-finite
// rows; a row with a NaN or +-inf coordinate lowers *bad_row to its index (when bad_row is given), so the caller can
// refuse the batch before it uses the codes.
__device__ __forceinline__ bool precedes(float a, int ia, float b, int ib) { return a < b || (a == b && ia < ib); }

template <typename code_t>
__global__ void encode_kernel(const float *__restrict__ x, const float *__restrict__ cb, code_t *__restrict__ codes,
                              int64_t N, int M, int Ks, int ds, unsigned long long *__restrict__ bad_row) {
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= N * M) return;
  const int64_t n = wid / M;
  const int m = (int)(wid - n * M);
  const float *v = x + n * (int64_t)M * ds + (int64_t)m * ds;
  if (bad_row) {
    bool bad = false;
    for (int j = lane; j < ds; j += 32) bad |= !isfinite(v[j]);
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMin(bad_row, (unsigned long long)n);
  }
  float best = CUDART_INF_F;
  int arg = 0x7fffffff;
  for (int c = lane; c < Ks; c += 32) {
    const float *w = cb + ((size_t)m * Ks + c) * ds;
    float acc = 0.f;
    for (int j = 0; j < ds; j++) {
      float t = __fsub_rn(v[j], w[j]);
      acc = __fadd_rn(acc, __fmul_rn(t, t));
    }
    if (isnan(acc)) acc = CUDART_INF_F;
    if (precedes(acc, c, best, arg)) {
      best = acc;
      arg = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ob = __shfl_xor_sync(0xffffffffu, best, o);
    int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (precedes(ob, oa, best, arg)) {
      best = ob;
      arg = oa;
    }
  }
  if (lane == 0) codes[n * M + m] = (code_t)arg;
}

}  // namespace

int launch_l2_normalize(annb_index *h, float *x, int64_t B, int D) {
  if (B == 0) return ANNB_OK;
  const int warps = 8;
  l2_normalize_kernel<<<(unsigned)((B + warps - 1) / warps), warps * 32, 0, h->stream>>>(x, B, D);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_adc_table(annb_index *h, const float *d_queries, int64_t B, float *d_out) {
  if (B == 0) return ANNB_OK;
  const int is_ip = h->metric != ANNB_METRIC_L2;
  const float bias = h->opt_ip_raw ? 0.f : (float)(1.0 / (double)h->Ks);
  const int chunks = (h->Ks + K1_THREADS - 1) / K1_THREADS;
  int64_t done = 0;
  while (done < B) {  // gridDim.y <= 65535
    int64_t nb = B - done;
    if (nb > (int64_t)65535 * K1_QT) nb = (int64_t)65535 * K1_QT;
    dim3 grid((unsigned)(h->M * chunks), (unsigned)((nb + K1_QT - 1) / K1_QT));
    const float *q = d_queries + done * h->dim;
    float *o = d_out + done * (int64_t)h->M * h->Ks;
    size_t sm_q = (size_t)K1_QT * h->ds * sizeof(float);
#define K1_CASE(DSV)                                                                                   \
  case DSV:                                                                                            \
    adc_table_kernel<DSV><<<grid, K1_THREADS, sm_q, h->stream>>>(q, h->d_codebook, o, nb, h->M, h->Ks, \
                                                                  h->ds, is_ip, bias, 1);              \
    break;
    switch (h->ds) {
      K1_CASE(2)
      K1_CASE(4)
      K1_CASE(6)
      K1_CASE(8)
      K1_CASE(12)
      K1_CASE(16)
      K1_CASE(24)
      K1_CASE(32)
      default: {
        // the query tile and the codewords in shared memory while they fit (ds <= 200 on H100), else neither
        size_t smb = sm_q + (size_t)K1_THREADS * (h->ds + 1) * sizeof(float);
        int optin = 0;
        ANNB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
        const int staged = smb <= (size_t)optin;
        if (!staged) smb = 0;
        if (smb > 48 * 1024)
          ANNB_CUDA(cudaFuncSetAttribute(adc_table_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb));
        adc_table_kernel<0><<<grid, K1_THREADS, smb, h->stream>>>(q, h->d_codebook, o, nb, h->M, h->Ks, h->ds,
                                                                 is_ip, bias, staged);
      }
    }
#undef K1_CASE
    h->launches++;
    ANNB_CUDA(cudaGetLastError());
    done += nb;
  }
  return ANNB_OK;
}

int launch_encode(annb_index *h, const float *d_x, int64_t n, void *d_codes, unsigned long long *d_bad_row) {
  if (n == 0) return ANNB_OK;
  const int warps = 8;
  int64_t total = n * h->M;
  unsigned grid = (unsigned)((total + warps - 1) / warps);
  if (d_bad_row) ANNB_CUDA(cudaMemsetAsync(d_bad_row, 0xff, sizeof(unsigned long long), h->stream));
  if (h->code_bytes == 1)
    encode_kernel<uint8_t><<<grid, warps * 32, 0, h->stream>>>(d_x, h->d_codebook, (uint8_t *)d_codes, n, h->M, h->Ks, h->ds,
                                                                d_bad_row);
  else
    encode_kernel<uint16_t><<<grid, warps * 32, 0, h->stream>>>(d_x, h->d_codebook, (uint16_t *)d_codes, n, h->M, h->Ks,
                                                                 h->ds, d_bad_row);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}
