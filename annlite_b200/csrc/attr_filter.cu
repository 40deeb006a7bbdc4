// attr_filter.cu -- attribute filters on the device.
//
// filter_eval_kernel turns a validated postfix program (include/annb.h, annb_filter_op_t) into the by-id bitmap the
// filtered walks read (hnsw_walk4f, hnsw_walk_flagged, the bitmap walk): one warp per 32 rows, one lane per row.
// The program and its constants sit in shared memory and every lane runs the same op on its own row, so control
// flow stays warp-uniform; the bool stack (<= ANNB_FILTER_MAX_DEPTH) is one register.  Column loads are coalesced
// 8-byte (INTEGER / FLOAT) or 4-byte (TEXT code) loads; validity and deletion words are one broadcast load per warp.
// Bytes moved: n * (sum of the widths of the referenced columns) + validity words + 2 * n / 8 (deleted in, bits out).
//
// filter_eval_kernel<true> evaluates F programs in the same pass (annb_filter_prepare_many): a warp runs them one after
// the other over its 32 rows, so HBM sees about one pass over the referenced columns plus F * n / 8 bytes of bitmaps.
//
// filter_compact_kernel turns a bitmap into the labels of its rows in internal-id order: per-block counts, one scan
// of the block counts (which also leaves the total behind them), then each block writes its rows at its offset.  An
// optional `drop` bitmap (the deletions) is masked out of every word on the way.
#include <algorithm>
#include <cstring>

#include "annb_internal.h"

namespace {

constexpr int kEvalThreads = 256;
constexpr int kCompactThreads = 256;  // one bitmap word per thread: 8192 rows per block

struct EvalCols {
  AttrColDev c[ANNB_MAX_ATTR_COLUMNS];
};

// index of the last element <= v in a[0, len) (0 if none); the step sequence depends on len only, so every lane of the
// warp runs the same iterations
template <typename T>
__device__ __forceinline__ bool sorted_contains(const T *a, int len, T v) {
  if (len <= 0) return false;
  int base = 0;
  while (len > 1) {
    const int half = len >> 1;
    base = (a[base + half] <= v) ? base + half : base;
    len -= half;
  }
  return a[base] == v;
}

// One program over the warp's 32 rows (row = w * 32 + lane): the bool the stack is left with.
__device__ __forceinline__ bool eval_program(const annb_filter_op_t *sprog, int n_ops, const uint8_t *cbytes,
                                             const EvalCols &cols, int64_t w, int64_t row, bool in, int lane) {
  uint32_t stack = 0;
  int sd = 0;
  for (int i = 0; i < n_ops; i++) {
    const annb_filter_op_t o = sprog[i];
    if (o.op == ANNB_FOP_AND || o.op == ANNB_FOP_OR) {
      sd--;
      const uint32_t a = (stack >> (sd - 1)) & 1u, b = (stack >> sd) & 1u;
      const uint32_t r = o.op == ANNB_FOP_AND ? (a & b) : (a | b);
      stack = (stack & ~(1u << (sd - 1))) | (r << (sd - 1));
      continue;
    }
    bool r;
    if (o.op == ANNB_FOP_FALSE) {
      r = false;
    } else if (o.op == ANNB_FOP_TRUE) {
      r = in;
    } else {
      const AttrColDev &c = cols.c[o.col];
      const bool valid = in && ((__ldg(c.valid + w) >> lane) & 1u);
      switch (o.op) {
        case ANNB_FOP_NOTNULL: r = valid; break;
        case ANNB_FOP_INT_RANGE:
        case ANNB_FOP_INT_NE:
        case ANNB_FOP_INT_IN:
        case ANNB_FOP_INT_NIN: {
          const int64_t v = valid ? __ldg(reinterpret_cast<const long long *>(c.vals) + row) : 0;
          const int64_t *k = reinterpret_cast<const int64_t *>(cbytes + o.a);
          if (o.op == ANNB_FOP_INT_RANGE) r = valid && k[0] <= v && v <= k[1];
          else if (o.op == ANNB_FOP_INT_NE) r = valid && v != k[0];
          else r = valid && (sorted_contains(k, o.b, v) == (o.op == ANNB_FOP_INT_IN));
          break;
        }
        case ANNB_FOP_FLT_RANGE:
        case ANNB_FOP_FLT_NE:
        case ANNB_FOP_FLT_IN:
        case ANNB_FOP_FLT_NIN: {
          const double v = valid ? __ldg(reinterpret_cast<const double *>(c.vals) + row) : 0.0;
          const double *k = reinterpret_cast<const double *>(cbytes + o.a);
          if (o.op == ANNB_FOP_FLT_RANGE) r = valid && k[0] <= v && v <= k[1];
          else if (o.op == ANNB_FOP_FLT_NE) r = valid && v != k[0];
          else r = valid && (sorted_contains(k, o.b, v) == (o.op == ANNB_FOP_FLT_IN));
          break;
        }
        default: {  // ANNB_FOP_CODE_IN
          const int32_t v = valid ? __ldg(reinterpret_cast<const int *>(c.vals) + row) : -1;
          const uint32_t *set = reinterpret_cast<const uint32_t *>(cbytes + o.a);
          r = valid && v >= 0 && v < o.b && ((set[v >> 5] >> (v & 31)) & 1u);
          break;
        }
      }
    }
    stack = (stack & ~(1u << sd)) | ((uint32_t)r << sd);
    sd++;
  }
  return stack & 1u;
}

// MULTI = false: one program (annb_filter_prepare).  MULTI = true: F programs over the same rows in one pass
// (annb_filter_prepare_many): the programs sit back to back in `prog` (program f = ops [offs[f], offs[f + 1]); their
// constant offsets already point into the one pool), a warp keeps its 32 rows and runs every program over them, so the
// column words the later programs read come from L1.  Program f writes the bitmap at bits + f * stride and adds its
// admitted rows to count[f].
template <bool MULTI>
__global__ void __launch_bounds__(kEvalThreads) filter_eval_kernel(const annb_filter_op_t *__restrict__ prog, int n_ops,
                                                                   const uint32_t *__restrict__ consts, int n_const_words,
                                                                   const EvalCols cols, int64_t n,
                                                                   const uint32_t *__restrict__ deleted,
                                                                   uint32_t *__restrict__ bits,
                                                                   unsigned long long *__restrict__ count, int F,
                                                                   const int *__restrict__ offs, int64_t stride) {
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ unsigned int block_count;
  annb_filter_op_t *sprog = reinterpret_cast<annb_filter_op_t *>(smem);
  uint32_t *sconst = smem + n_ops * 4;  // sizeof(annb_filter_op_t) == 16: the pool stays 16-byte aligned
  const uint32_t *gprog = reinterpret_cast<const uint32_t *>(prog);
  for (int i = threadIdx.x; i < n_ops * 4; i += blockDim.x) smem[i] = gprog[i];
  for (int i = threadIdx.x; i < n_const_words; i += blockDim.x) sconst[i] = consts[i];
  // MULTI: [F + 1 program offsets][F block counts] behind the pool
  int *soff = reinterpret_cast<int *>(sconst + n_const_words);
  unsigned int *scount = reinterpret_cast<unsigned int *>(soff + F + 1);
  if constexpr (MULTI) {
    for (int i = threadIdx.x; i <= F; i += blockDim.x) soff[i] = offs[i];
    for (int i = threadIdx.x; i < F; i += blockDim.x) scount[i] = 0;
  }
  if (threadIdx.x == 0) block_count = 0;
  __syncthreads();
  const uint8_t *cbytes = reinterpret_cast<const uint8_t *>(sconst);

  const int lane = threadIdx.x & 31;
  const int64_t words = (n + 31) / 32 + 1;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  unsigned int mine = 0;
  for (int64_t w = (((int64_t)blockIdx.x * blockDim.x) + threadIdx.x) >> 5; w < words; w += nwarps) {
    const int64_t row = w * 32 + lane;
    const bool in = row < n;
    if constexpr (MULTI) {
      const bool live = in && !(deleted && ((__ldg(deleted + w) >> lane) & 1u));
      for (int f = 0; f < F; f++) {
        const int o0 = soff[f];
        const bool r = eval_program(sprog + o0, soff[f + 1] - o0, cbytes, cols, w, row, in, lane);
        const bool keep = live && r;
        const uint32_t word = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) {
          bits[f * stride + w] = word;
          if (word) atomicAdd(&scount[f], (unsigned int)__popc(word));
        }
      }
    } else {
      const bool r = eval_program(sprog, n_ops, cbytes, cols, w, row, in, lane);
      const bool keep = in && r && !(deleted && ((__ldg(deleted + w) >> lane) & 1u));
      const uint32_t word = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) {
        bits[w] = word;
        mine += __popc(word);
      }
    }
  }
  if constexpr (MULTI) {
    __syncthreads();
    for (int i = threadIdx.x; i < F; i += blockDim.x)
      if (scount[i]) atomicAdd(count + i, (unsigned long long)scount[i]);
  } else {
    if (lane == 0 && mine) atomicAdd(&block_count, mine);
    __syncthreads();
    if (threadIdx.x == 0 && block_count) atomicAdd(count, (unsigned long long)block_count);
  }
}

__device__ __forceinline__ unsigned int block_exclusive_scan(unsigned int v, unsigned int *warp_sums, unsigned int *total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    const int nw = blockDim.x >> 5;
    unsigned int s = lane < nw ? warp_sums[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) warp_sums[lane] = s;  // inclusive sums of the warps
  }
  __syncthreads();
  const unsigned int before = wid ? warp_sums[wid - 1] : 0u;
  if (total) *total = warp_sums[(blockDim.x >> 5) - 1];
  return before + x - v;
}

__device__ __forceinline__ uint32_t listed_word(const uint32_t *bits, const uint32_t *drop, int64_t w, int64_t nwords) {
  return w < nwords ? bits[w] & ~(drop ? drop[w] : 0u) : 0u;
}

// pass 1: admitted rows per block
__global__ void __launch_bounds__(kCompactThreads) filter_count_kernel(const uint32_t *__restrict__ bits,
                                                                       const uint32_t *__restrict__ drop, int64_t nwords,
                                                                       unsigned int *__restrict__ block_counts) {
  __shared__ unsigned int warp_sums[kCompactThreads / 32];
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int c = __popc(listed_word(bits, drop, w, nwords));
  unsigned int total;
  block_exclusive_scan(c, warp_sums, &total);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = total;
}

// pass 2: exclusive scan of the block counts, in place (one block); the total goes to block_counts[nblocks]
__global__ void __launch_bounds__(1024) filter_scan_kernel(unsigned int *__restrict__ block_counts, int64_t nblocks) {
  __shared__ unsigned int warp_sums[32];
  __shared__ unsigned int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < nblocks; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const unsigned int v = i < nblocks ? block_counts[i] : 0u;
    unsigned int total;
    const unsigned int ex = block_exclusive_scan(v, warp_sums, &total);
    if (i < nblocks) block_counts[i] = carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) block_counts[nblocks] = carry;
}

// pass 3: each block writes the labels of its admitted rows at its offset, in internal-id order
__global__ void __launch_bounds__(kCompactThreads) filter_compact_kernel(const uint32_t *__restrict__ bits,
                                                                         const uint32_t *__restrict__ drop, int64_t nwords,
                                                                         const unsigned int *__restrict__ block_offsets,
                                                                         const uint64_t *__restrict__ labels,
                                                                         uint64_t *__restrict__ out) {
  __shared__ unsigned int warp_sums[kCompactThreads / 32];
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t word = listed_word(bits, drop, w, nwords);
  unsigned int pos = block_offsets[blockIdx.x] + block_exclusive_scan(__popc(word), warp_sums, nullptr);
  while (word) {
    const int b = __ffs(word) - 1;
    word &= word - 1;
    out[pos++] = labels[w * 32 + b];
  }
}

// per-query filter batches: one warp per row, a lane per 4-byte word
__global__ void __launch_bounds__(256) rows_copy_kernel(const uint32_t *__restrict__ src, uint32_t *__restrict__ dst,
                                                        const uint32_t *__restrict__ idx, int64_t n, int row_words,
                                                        bool scatter) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  const int64_t r = __ldg(idx + i);
  const uint32_t *s = src + (scatter ? i : r) * row_words;
  uint32_t *d = dst + (scatter ? r : i) * row_words;
  for (int j = threadIdx.x & 31; j < row_words; j += 32) d[j] = s[j];
}

}  // namespace

int launch_rows_copy(annb_index *h, const void *src, void *dst, const uint32_t *d_idx, int64_t n, int row_words, bool scatter) {
  if (n == 0) return ANNB_OK;
  rows_copy_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, h->stream>>>((const uint32_t *)src, (uint32_t *)dst, d_idx, n,
                                                                            row_words, scatter);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_filter_eval(annb_index *h, const annb_filter_op_t *d_prog, int n_ops, const void *d_consts, int n_const_bytes,
                       const AttrColDev *cols, int n_cols, int64_t n, const uint32_t *d_deleted, uint32_t *d_bits,
                       unsigned long long *d_count) {
  EvalCols ec;
  memset(&ec, 0, sizeof(ec));
  for (int i = 0; i < n_cols && i < ANNB_MAX_ATTR_COLUMNS; i++) ec.c[i] = cols[i];
  const int64_t words = (n + 31) / 32 + 1;
  const int64_t want = (words * 32 + kEvalThreads - 1) / kEvalThreads;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)h->sm_count * 8));
  const size_t smem = (size_t)n_ops * sizeof(annb_filter_op_t) + (size_t)n_const_bytes;
  filter_eval_kernel<false><<<blocks, kEvalThreads, smem, h->stream>>>(d_prog, n_ops, (const uint32_t *)d_consts, n_const_bytes / 4,
                                                                       ec, n, d_deleted, d_bits, d_count, 1, nullptr, 0);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_filter_eval_many(annb_index *h, int F, const annb_filter_op_t *d_prog, const int *d_offs, int n_ops,
                            const void *d_consts, int n_const_bytes, const AttrColDev *cols, int n_cols, int64_t n,
                            const uint32_t *d_deleted, uint32_t *d_bits, int64_t stride_words,
                            unsigned long long *d_counts) {
  EvalCols ec;
  memset(&ec, 0, sizeof(ec));
  for (int i = 0; i < n_cols && i < ANNB_MAX_ATTR_COLUMNS; i++) ec.c[i] = cols[i];
  const int64_t words = (n + 31) / 32 + 1;
  const int64_t want = (words * 32 + kEvalThreads - 1) / kEvalThreads;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)h->sm_count * 8));
  const size_t smem = (size_t)n_ops * sizeof(annb_filter_op_t) + (size_t)n_const_bytes + (size_t)(2 * F + 1) * 4;
  if (smem > 48 * 1024)
    ANNB_CUDA(cudaFuncSetAttribute(filter_eval_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  filter_eval_kernel<true><<<blocks, kEvalThreads, smem, h->stream>>>(d_prog, n_ops, (const uint32_t *)d_consts, n_const_bytes / 4,
                                                                      ec, n, d_deleted, d_bits, d_counts, F, d_offs, stride_words);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int64_t filter_compact_blocks(int64_t n) {
  const int64_t nwords = (n + 31) / 32;
  return std::max<int64_t>(1, (nwords + kCompactThreads - 1) / kCompactThreads);
}

int launch_filter_count(annb_index *h, const uint32_t *d_bits, const uint32_t *d_drop, int64_t n, unsigned int *d_block_scratch) {
  const int64_t nb = filter_compact_blocks(n);
  filter_count_kernel<<<(unsigned)nb, kCompactThreads, 0, h->stream>>>(d_bits, d_drop, (n + 31) / 32, d_block_scratch);
  filter_scan_kernel<<<1, 1024, 0, h->stream>>>(d_block_scratch, nb);
  h->launches += 2;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_filter_compact(annb_index *h, const uint32_t *d_bits, const uint32_t *d_drop, int64_t n, const uint64_t *d_labels,
                          uint64_t *d_out, const unsigned int *d_block_scratch) {
  filter_compact_kernel<<<(unsigned)filter_compact_blocks(n), kCompactThreads, 0, h->stream>>>(d_bits, d_drop, (n + 31) / 32,
                                                                                              d_block_scratch, d_labels, d_out);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}
