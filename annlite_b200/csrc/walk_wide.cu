// walk_wide.cu -- hnsw_walk_wide: the HNSW walk for PQ code rows wider than 128 bytes (sm_90a).
//
// Semantics are hnsw_walk_general's (hnsw_search.cu): searchKnn (hnswalg.h:1237-1295) and searchKnnWithFilter
// (:1297-1361) followed literally, one warp per query, with the candidate bag in shared memory (spilling to per-warp
// global scratch), an exact visited bitmap in per-warp global scratch, and the same admission rules for deletions, a
// by-id filter bitmap or one bitmap per query (SearchParams::query_filter).  One lane scores one neighbour.
//
// What differs is where a distance comes from.  At M = 768 one query's ADC table is M x Ks x 4 = 786 KB: it never
// fits in shared memory, and a (B, M, Ks) array of them would be 7.9 GB for 10 000 queries.  So no table is built.
// For each neighbour and each m in order the lane computes the table entry K1 would have written -- the same
// __fsub_rn / __fmul_rn / __fadd_rn sequence over j as adc_table_kernel, and the IP epilogue bias - ip -- from the
// query (staged in shared memory) and the codebook (D x Ks x 4 bytes for any M, L2 resident), then adds it to the
// running sum sequentially over m, as PQLookup does (space_pq.h:30-35).  Every term is bit-equal to K1's entry, so
// every distance is bit-equal to the table walk's.  Given tables (the literal dtables call form) the same kernel
// reads them instead.
//
// Layout (annb_internal.h, WideDev): level-0 records are [maxM0 x u32 node id]; every node's code row is stored once
// in a by-id matrix with 16-byte aligned rows; upper records carry their links' node ids so the descent can reach
// the codes.  The entry node's code is read from the matrix.
#include <math_constants.h>

#include <algorithm>

#include "annb_internal.h"
#include "walk_common.cuh"

namespace {

constexpr int WIDE_WARPS = 8;

// what one distance needs: the query (or the query's table) and the codebook
struct Scorer {
  const float *x;    // the query (shared memory, or global when it does not fit), nullptr when T is given
  const float *T;    // the query's (M, Ks) table, or nullptr
  const float *cb;   // (M, Ks, ds)
  int M, Ks, ds, is_ip;
  float bias;
};

// adc_table_kernel's entry T[m][c]: sequential over j, every operation rounded separately
__device__ __forceinline__ float table_entry(const Scorer &s, int m, uint32_t c) {
  const float *w = s.cb + ((size_t)m * s.Ks + c) * s.ds;
  const float *x = s.x + (size_t)m * s.ds;
  float acc = 0.f;
  if (s.is_ip) {
    for (int j = 0; j < s.ds; j++) acc = __fadd_rn(acc, __fmul_rn(__ldg(w + j), x[j]));
    acc = __fsub_rn(s.bias, acc);
  } else {
    for (int j = 0; j < s.ds; j++) {
      const float t = __fsub_rn(__ldg(w + j), x[j]);
      acc = __fadd_rn(acc, __fmul_rn(t, t));
    }
  }
  return acc;
}

// PQLookup over one code row (16-byte aligned; the bytes past M * CB up to the row stride are never used)
template <int CB>
__device__ __forceinline__ float score_row(const Scorer &s, const uint8_t *row) {
  float r = 0.f;
  const int bytes = s.M * CB;
  for (int b0 = 0; b0 < bytes; b0 += 16) {
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(row + b0));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 16 / CB; i++) {
      const int m = b0 / CB + i;
      if (m < s.M) {
        const uint32_t c = CB == 1 ? (w[i >> 2] >> (8 * (i & 3))) & 0xffu : (w[i >> 1] >> (16 * (i & 1))) & 0xffffu;
        r = __fadd_rn(r, s.T ? __ldg(s.T + (size_t)m * s.Ks + c) : table_entry(s, m, c));
      }
    }
  }
  return r;
}

// PQF: the bitmap of query row q is p.query_filter[q] (nullptr = "not deleted"); q_smem: the query is staged in
// shared memory (else read from global)
template <int EPL, int CB, bool PQF>
__global__ void __launch_bounds__(WIDE_WARPS * 32) hnsw_walk_wide(const GraphDev g, const SearchParams p, const WideDev wd,
                                                                  const int has_del, const int q_smem) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int D = wd.dim;
  const int qfloats = q_smem ? (D + 3) / 4 * 4 : 0;
  // [nwarps x query] [nwarps x (32*EPL merge scratch + SBAG bag) x 8 B]
  float *xs = reinterpret_cast<float *>(smem_raw) + (size_t)warp * qfloats;
  uint2 *scratch = reinterpret_cast<uint2 *>(smem_raw + (size_t)nwarps * qfloats * 4) + (size_t)warp * (32 * EPL + SBAG);
  uint64_t *sbag = reinterpret_cast<uint64_t *>(scratch + 32 * EPL);
  const unsigned lt_mask = (1u << lane) - 1u;
  const int ef = p.ef;
  const int64_t slot = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  uint32_t *vis = p.visited + slot * p.visited_words;
  uint32_t *touched = p.touched + slot * (int64_t)p.touched_cap;
  uint64_t *gbag = p.cand + slot * (int64_t)p.cand_cap;
  const uint32_t *filter = p.filter;
  bool use_filter = filter != nullptr;
  Scorer s;
  s.cb = wd.codebook;
  s.M = g.M;
  s.Ks = g.Ks;
  s.ds = p.ds;
  s.is_ip = p.is_ip;
  s.bias = p.bias;
  const uint8_t *codes = wd.codes;
  const int64_t stride = wd.code_stride;

  for (;;) {
    const int64_t wi = next_query(p.work_counter, lane);
    if (wi >= p.B) break;
    const int64_t q = p.qmap ? (int64_t)__ldg(p.qmap + wi) : wi;
    if constexpr (PQF) {
      filter = p.query_filter[q];
      use_filter = filter != nullptr;
    }
    if (p.tables) {
      s.T = p.tables + q * (int64_t)g.M * g.Ks;
      s.x = nullptr;
    } else {
      s.T = nullptr;
      if (q_smem) {
        __syncwarp();
        for (int i = lane; i < D; i += 32) xs[i] = __ldg(p.queries + q * D + i);
        __syncwarp();
        s.x = xs;
      } else {
        s.x = p.queries + q * D;
      }
    }

    // greedy descent maxlevel..1 (hnswalg.h:1245-1274): the first minimum among neighbours that beat curdist
    int hops = 0, nbrs = 0, evals = 1;
    float cur = score_row<CB>(s, codes + (size_t)g.ep_node * stride);  // dist to the entry point (:1246)
    uint32_t rec = g.ep_rec;
    for (int level = g.maxlevel; level > 0; level--) {
      const uint8_t *base = g.up + g.up_off[level];
      bool changed = true;
      while (changed) {
        changed = false;
        const uint8_t *r = base + (size_t)rec * g.recu_bytes;
        float best = cur;
        uint32_t best_link = EMPTY_LINK;
        hops++;
        for (int c0 = 0; c0 < g.maxM; c0 += 32) {
          const int j = c0 + lane;
          const uint32_t link = j < g.maxM ? __ldg(reinterpret_cast<const uint32_t *>(r) + j) : EMPTY_LINK;
          const bool valid = link != EMPTY_LINK;
          float d = CUDART_INF_F;
          if (valid) {
            const uint32_t node = __ldg(reinterpret_cast<const uint32_t *>(r + g.code_offu) + j);
            d = score_row<CB>(s, codes + (size_t)node * stride);
          }
          const int nv = __popc(__ballot_sync(FULL_MASK, valid));
          nbrs += nv;
          evals += nv;
          float md = d;
          int mj = lane;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(FULL_MASK, md, o);
            const int oj = __shfl_xor_sync(FULL_MASK, mj, o);
            if (od < md || (od == md && oj < mj)) {
              md = od;
              mj = oj;
            }
          }
          if (md < best) {
            best = md;
            best_link = __shfl_sync(FULL_MASK, link, mj);
          }
          if (nv < 32) break;
        }
        if (best_link != EMPTY_LINK) {
          cur = best;
          rec = best_link;
          changed = true;
        }
      }
      rec = __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)rec * g.recu_bytes + g.tail_offu) + 1);
    }

    WarpList<EPL> L;  // top_candidates: admitted entries only
    L.clear();
    int topsize = 0, ns = 0, ng = 0, ntouched = 0;
    bool overflow = false;
    float lower;
    {
      const uint32_t ep = rec;
      bool ok;
      if (use_filter) ok = (filter[ep >> 5] >> (ep & 31)) & 1u;                    // :353-354
      else ok = !has_del || !((g.deleted[ep >> 5] >> (ep & 31)) & 1u);             // :254
      if (ok) {
        evals++;
        lower = cur;
        L.insert(cur, ep, ef);
        topsize = 1;
        if (lane == 0) sbag[0] = pack_cand(cur, ep);
      } else {
        lower = 3.402823466e+38f;  // std::numeric_limits<float>::max()
        if (lane == 0) sbag[0] = pack_cand(lower, ep);
      }
      ns = 1;
      if (lane == 0) {
        vis[ep >> 5] |= 1u << (ep & 31);
        touched[0] = ep;
      }
      ntouched = 1;
      __syncwarp();
    }

    while (ns + ng > 0) {
      // candidate_set.top(): nearest candidate (shared part, then the spilled part)
      float bd = CUDART_INF_F;
      int bi = 0x7fffffff;
      uint32_t bid = 0;
      for (int i = lane; i < ns; i += 32) {
        const uint64_t c = sbag[i];
        const float d = cand_d(c);
        if (d < bd || (d == bd && i < bi)) {
          bd = d;
          bi = i;
          bid = cand_id(c);
        }
      }
      for (int i = lane; i < ng; i += 32) {
        const uint64_t c = gbag[i];
        const float d = cand_d(c);
        if (d < bd || (d == bd && i + SBAG < bi)) {
          bd = d;
          bi = i + SBAG;
          bid = cand_id(c);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(FULL_MASK, bd, o);
        const int oi = __shfl_xor_sync(FULL_MASK, bi, o);
        const uint32_t oid = __shfl_xor_sync(FULL_MASK, bid, o);
        if (od < bd || (od == bd && oi < bi)) {
          bd = od;
          bi = oi;
          bid = oid;
        }
      }
      if (use_filter) {
        if (bd > lower) break;                                                     // :371
      } else if (bd > lower && (topsize == ef || !has_del)) {
        break;                                                                     // :270
      }
      const uint32_t *rec0 = reinterpret_cast<const uint32_t *>(g.rec0 + (size_t)bid * g.rec0_bytes);
      const uint32_t link0 = (lane < g.maxM0) ? __ldg(rec0 + lane) : EMPTY_LINK;
      if (lane == 0) {
        if (bi < SBAG) sbag[bi] = sbag[ns - 1];
        else gbag[bi - SBAG] = gbag[ng - 1];
      }
      if (bi < SBAG) ns--;
      else ng--;
      __syncwarp();
      // candidates beyond lowerBound are dead once top is full (lowerBound only falls): drop them now and then
      if (topsize == ef && ((hops & 3) == 3 || ns > SBAG - 40)) {
        int wpos = 0;
        for (int b0 = 0; b0 < ns; b0 += 32) {
          const int i = b0 + lane;
          uint64_t c = 0;
          bool keep = false;
          if (i < ns) {
            c = sbag[i];
            keep = !(cand_d(c) > lower);
          }
          const unsigned km = __ballot_sync(FULL_MASK, keep);
          __syncwarp();
          if (keep) sbag[wpos + __popc(km & lt_mask)] = c;
          wpos += __popc(km);
          __syncwarp();
        }
        ns = wpos;
        if (ng > 0) {
          wpos = 0;
          for (int b0 = 0; b0 < ng; b0 += 32) {
            const int i = b0 + lane;
            uint64_t c = 0;
            bool keep = false;
            if (i < ng) {
              c = gbag[i];
              keep = !(cand_d(c) > lower);
            }
            const unsigned km = __ballot_sync(FULL_MASK, keep);
            __syncwarp();
            if (keep) gbag[wpos + __popc(km & lt_mask)] = c;
            wpos += __popc(km);
            __syncwarp();
          }
          ng = wpos;
        }
      }

      hops++;
      for (int c0 = 0; c0 < g.maxM0; c0 += 32) {
        const int j = c0 + lane;
        const uint32_t link = (c0 == 0) ? link0 : (j < g.maxM0 ? __ldg(rec0 + j) : EMPTY_LINK);
        const bool valid = link != EMPTY_LINK;
        const int nv = __popc(__ballot_sync(FULL_MASK, valid));
        nbrs += nv;
        bool fresh = false;
        if (valid) {
          const uint32_t bit = 1u << (link & 31);
          const uint32_t old = atomicOr(vis + (link >> 5), bit);  // exact visited set (:299-301)
          fresh = !(old & bit);
        }
        const unsigned fmask = __ballot_sync(FULL_MASK, fresh);
        const int nf = __popc(fmask);
        evals += nf;
        if (fresh) {
          const int o = ntouched + __popc(fmask & lt_mask);
          if (o < p.touched_cap) touched[o] = link;
        }
        ntouched += nf;
        if (ntouched > p.touched_cap) overflow = true;
        float d = CUDART_INF_F;
        bool admit = false;
        if (fresh) {
          d = score_row<CB>(s, codes + (size_t)link * stride);
          if (use_filter) admit = (filter[link >> 5] >> (link & 31)) & 1u;        // :423-426
          else admit = !has_del || !((g.deleted[link >> 5] >> (link & 31)) & 1u);  // :314
        }
        // admission for the whole neighbour list at once (hnsw_search.cu: hnsw_walk_general has the argument)
        const bool cand_ok = fresh && (topsize < ef || lower > d);
        const unsigned cmask = __ballot_sync(FULL_MASK, cand_ok);
        if (cmask) {
          const int cnt = __popc(cmask);
          const int r = __popc(cmask & lt_mask);
          if (ns + cnt <= SBAG) {
            if (cand_ok) sbag[ns + r] = pack_cand(d, link);
            ns += cnt;
          } else {
            if (cand_ok && ng + r < p.cand_cap) gbag[ng + r] = pack_cand(d, link);
            if (ng + cnt > p.cand_cap) overflow = true;
            ng = min(ng + cnt, p.cand_cap);
          }
          float unused_worst;
          L.merge(d, link, cand_ok && admit, ef, scratch, topsize, unused_worst, ID_MASK);
          if (topsize > 0) lower = L.key_at(topsize - 1);                         // :320-321
        }
        __syncwarp();
        if (nv < 32) break;
      }
    }
    // reset the visited bits this query set
    __syncwarp();
    {
      const int nt = min(ntouched, p.touched_cap);
      for (int i = lane; i < nt; i += 32) vis[touched[i] >> 5] = 0u;
      if (ntouched > p.touched_cap) {
        for (int64_t i = lane; i < p.visited_words; i += 32) vis[i] = 0u;
      }
    }
    if (overflow && lane == 0) atomicExch(p.overflow_flag, 1);
    __syncwarp();
    write_results<EPL>(g, p, q, L, lane, hops, nbrs, evals);
  }
}

template <int EPL, int CB, bool PQF>
int launch_wide_t(annb_index *h, const SearchParams &p_in) {
  SearchParams p = p_in;
  // the K1 form of the table entries (launch_adc_table)
  p.ds = h->ds;
  p.is_ip = h->metric != ANNB_METRIC_L2;
  p.bias = h->opt_ip_raw ? 0.f : (float)(1.0 / (double)h->Ks);
  WideDev wd;
  wd.codes = h->d_wide_codes;
  wd.codebook = h->d_codebook;
  wd.code_stride = wide_code_stride(h);
  wd.dim = h->dim;
  if (!p.tables && !wd.codebook) ANNB_FAIL(ANNB_ESTATE, "Please train the PQ before using HNSW quantization backend");
  auto kern = hnsw_walk_wide<EPL, CB, PQF>;
  int optin = 0;
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device);
  const size_t bag = (size_t)(32 * EPL + SBAG) * sizeof(uint2), qbytes = (size_t)(h->dim + 3) / 4 * 4 * sizeof(float);
  const int warps = WIDE_WARPS, threads = warps * 32;
  int q_smem = !p.tables && warps * (qbytes + bag) <= (size_t)optin;  // very long vectors: the query stays in global memory
  const size_t smem = warps * ((q_smem ? qbytes : 0) + bag);
  if (smem > 48 * 1024) ANNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0;
  ANNB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
  if (occ < 1) ANNB_FAIL(ANNB_ELIMIT, "hnsw_walk_wide does not fit on this device (registers/shared memory)");
  ANNB_TRY_RC(walk_counter(h, p));
  const int blocks = (int)std::min<int64_t>((int64_t)h->sm_count * occ, (p.B + warps - 1) / warps);
  const int has_del = h->g.num_deleted > 0 ? 1 : 0;
  return run_bitmap_walk(h, p, blocks, warps, "wide", [&](int b, const SearchParams &pr) {
    kern<<<b, threads, smem, h->stream>>>(h->gd, pr, wd, has_del, q_smem);
  });
}

template <int EPL>
int launch_wide_e(annb_index *h, const SearchParams &p) {
  const bool pqf = p.query_filter != nullptr;
  if (h->code_bytes == 1) return pqf ? launch_wide_t<EPL, 1, true>(h, p) : launch_wide_t<EPL, 1, false>(h, p);
  return pqf ? launch_wide_t<EPL, 2, true>(h, p) : launch_wide_t<EPL, 2, false>(h, p);
}

}  // namespace

int launch_walk_wide(annb_index *h, const SearchParams &p) {
  if (p.B == 0) return ANNB_OK;
  if (!h->d_wide_codes || h->gd.n == 0) ANNB_FAIL(ANNB_ESTATE, "internal: the wide device graph is not built");
  return with_epl(p.ef, [&](auto epl) { return launch_wide_e<decltype(epl)::value>(h, p); });
}
