// hnsw_search.cu -- K3: warp-per-query HNSW walk over PQ codes (sm_90a).
//
// Reference semantics: HierarchicalNSW::searchKnn (include/hnswlib/hnswalg.h:1237-1295) =
// greedy descent on levels maxlevel..1 (:1248-1274) + searchBaseLayerST (:243-329), and the
// filtered twin searchKnnWithFilter (:1297-1361) + searchBaseLayerSTWithFilter (:332-440), with
// the PQ distance PQLookup (include/hnswlib/space_pq.h:16-37): d = sum_m T[m][code_m], m
// sequential from 0.f -- one lane scores one neighbour, so the fp32 sum order is the reference's.
//
// Kernels:
//  * hnsw_walk_fast     -- no deletions, no filter, maxM0 <= 32 (the headline path).  The reference's two
//    heaps collapse into ONE sorted list of ef entries (registers + a shared-memory mirror): without
//    deletions every candidate is also a top-candidate, so the candidate heap is exactly the not-yet-
//    expanded members of the list (a candidate evicted from top_candidates has d >= lowerBound and the
//    loop would break before expanding it, :270).  No visited set is needed either: a re-encountered
//    node is either still in the list (dropped by an id compare restricted to equal keys) or was
//    rejected / evicted with d >= lowerBound, and lowerBound only falls once the list is full, so it is
//    rejected again (:306).  The walk therefore WRITES NOTHING to global memory until its k results.
//    Per hop: score all <= 32 neighbours (one lane each), rank the admitted ones by a branch-free
//    binary search over the mirror, request the likely next node's record (overlaps the merge), merge
//    by rank counting + scatter through the mirror, then read the true next node off the merged list.
//    Differences from the reference are confined to exact fp32 distance ties.
//  * hnsw_walk_chunked  -- same semantics for graphs with maxM0 > 32 (neighbour list in 32-wide chunks,
//    WarpList::merge per chunk, no prefetch).
//  * hnsw_walk_general  -- deletions and/or filter: follows the reference literally with a separate
//    candidate bag (shared memory, spilling to per-warp global scratch) and an exact visited bitmap
//    (per-warp global scratch, L2 resident), because nodes that fail the filter are traversed but never
//    admitted, so the single-list argument above does not hold.
//
// Memory layout (DESIGN.md section 3): node record = [maxM0 links][maxM0 neighbour codes], so one
// hop is one contiguous, coalesced read (384 B for M=8) instead of an adjacency read followed by
// up to 32 dependent 8-byte gathers.  The per-query table (M*Ks fp32) is staged into shared memory
// by one TMA bulk copy (cp.async.bulk + mbarrier) per query.  Only two-byte codes have a table too big
// for shared memory (large Ks): hnsw_walk_fast / _chunked / _general then read it from global memory
// (SMEM_TABLE = false).  One-byte codes are compiled in the shared-memory form only (launch_walk).
#include <math_constants.h>

#include <algorithm>

#include "annb_internal.h"
#include "tma_utils.cuh"
#include "walk_common.cuh"

namespace {

constexpr uint32_t EXPANDED_BIT = 0x80000000u;

// ---- code row in registers -------------------------------------------------------------------
template <int CR>
struct CodeWords {
  uint32_t w[CR / 4];
  __device__ __forceinline__ void load(const uint8_t *p) {
    if (CR == 4) {
      w[0] = __ldg(reinterpret_cast<const uint32_t *>(p));
    } else if (CR == 8) {
      uint2 t = __ldg(reinterpret_cast<const uint2 *>(p));
      w[0] = t.x;
      w[1] = t.y;
    } else {
#pragma unroll
      for (int i = 0; i < CR / 16; i++) {
        uint4 t = __ldg(reinterpret_cast<const uint4 *>(p) + i);
        w[4 * i + 0] = t.x;
        w[4 * i + 1] = t.y;
        w[4 * i + 2] = t.z;
        w[4 * i + 3] = t.w;
      }
    }
  }
};

// PQLookup (space_pq.h:30-35): strictly sequential fp32 sum over subquantisers
template <int CR, int CB>
__device__ __forceinline__ float pq_lookup(const float *T, const CodeWords<CR> &c, int Ks) {
  float r = 0.f;
  constexpr int M = CR / CB;
#pragma unroll
  for (int m = 0; m < M; m++) {
    uint32_t code;
    if (CB == 1) code = (c.w[m >> 2] >> (8 * (m & 3))) & 0xffu;
    else code = (c.w[m >> 1] >> (16 * (m & 1))) & 0xffffu;
    r = __fadd_rn(r, T[m * Ks + code]);
  }
  return r;
}
// generic: code bytes straight from memory
template <int CB>
__device__ __forceinline__ float pq_lookup_mem(const float *T, const uint8_t *p, int M, int Ks) {
  float r = 0.f;
  for (int m = 0; m < M; m++) {
    uint32_t code = CB == 1 ? (uint32_t)p[m] : (uint32_t)reinterpret_cast<const uint16_t *>(p)[m];
    r = __fadd_rn(r, T[m * Ks + code]);
  }
  return r;
}

template <int CR, int CB>
__device__ __forceinline__ float score(const float *T, const uint8_t *code_ptr, int M, int Ks) {
  if (CR > 0) {
    CodeWords<(CR > 0 ? CR : 4)> c;
    c.load(code_ptr);
    return pq_lookup<(CR > 0 ? CR : 4), CB>(T, c, Ks);
  } else {
    return pq_lookup_mem<CB>(T, code_ptr, M, Ks);
  }
}

__device__ __forceinline__ void load_table(float *dst, const float *__restrict__ src, int TS, int lane) {
  if ((TS & 3) == 0) {
    const float4 *s4 = reinterpret_cast<const float4 *>(src);
    float4 *d4 = reinterpret_cast<float4 *>(dst);
    for (int i = lane; i < (TS >> 2); i += 32) d4[i] = __ldg(s4 + i);
  } else {
    for (int i = lane; i < TS; i += 32) dst[i] = __ldg(src + i);
  }
}

struct Walk {
  uint32_t node;   // node reached on level 0
  float dist;      // its distance
  int hops, nbrs, evals;
};

// Greedy descent maxlevel..1 (hnswalg.h:1245-1274).  After scanning one node's list the
// reference holds the FIRST minimum among neighbours that beat curdist (strict <, sequential).
template <int CR, int CB>
__device__ __forceinline__ Walk descend(const GraphDev &g, const float *T, int lane) {
  Walk w;
  w.hops = 0;
  w.nbrs = 0;
  w.evals = 1;
  w.dist = pq_lookup_mem<CB>(T, g.ep_code, g.M, g.Ks);  // dist to the entry point (:1246)
  uint32_t rec = g.ep_rec;
  for (int level = g.maxlevel; level > 0; level--) {
    const uint8_t *base = g.up + g.up_off[level];
    bool changed = true;
    while (changed) {
      changed = false;
      const uint8_t *r = base + (size_t)rec * g.recu_bytes;
      float best = w.dist;
      uint32_t best_link = EMPTY_LINK;
      w.hops++;
      for (int c0 = 0; c0 < g.maxM; c0 += 32) {
        const int j = c0 + lane;
        uint32_t link = j < g.maxM ? __ldg(reinterpret_cast<const uint32_t *>(r) + j) : EMPTY_LINK;
        const bool valid = link != EMPTY_LINK;
        float d = CUDART_INF_F;
        if (valid) d = score<CR, CB>(T, r + g.code_offu + (size_t)j * g.code_row, g.M, g.Ks);
        const int nv = __popc(__ballot_sync(FULL_MASK, valid));
        w.nbrs += nv;
        w.evals += nv;
        // warp argmin, first index wins ties
        float md = d;
        int mj = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          float od = __shfl_xor_sync(FULL_MASK, md, o);
          int oj = __shfl_xor_sync(FULL_MASK, mj, o);
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
        w.dist = best;
        rec = best_link;
        changed = true;
      }
    }
    // step down: record index on the level below (node id when level == 1)
    rec = __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)rec * g.recu_bytes + g.tail_offu) + 1);
  }
  w.node = rec;
  return w;
}

// =================================================================================================
// fast path: no deletions, no filter
// =================================================================================================
template <int EPL, int CR, int CB, bool SMEM_TABLE>
__global__ void hnsw_walk_chunked(const GraphDev g, const SearchParams p, const int table_stride_bytes) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int TS = g.M * g.Ks;
  // [nwarps x table (SMEM_TABLE only)] [nwarps x 32*EPL uint2 merge scratch]
  float *Ts = reinterpret_cast<float *>(smem_raw + (size_t)warp * table_stride_bytes);
  uint2 *scratch = reinterpret_cast<uint2 *>(smem_raw + (size_t)nwarps * table_stride_bytes) + (size_t)warp * 32 * EPL;
  const int ef = p.ef;

  for (;;) {
    const int64_t q = next_query(p.work_counter, lane);
    if (q >= p.B) break;
    const float *T;
    if (SMEM_TABLE) {
      __syncwarp();
      load_table(Ts, p.tables + q * TS, TS, lane);
      __syncwarp();
      T = Ts;
    } else {
      T = p.tables + q * TS;
    }

    Walk w = descend<CR, CB>(g, T, lane);
    int hops = w.hops, nbrs = w.nbrs, evals = w.evals + 1;  // searchBaseLayerST re-scores the entry (:255)

    WarpList<EPL> L;
    L.clear();
    int size = 0;
    float worst = CUDART_INF_F;  // lowerBound; +inf while the list is not full (:306)
    L.merge(w.dist, w.node, lane == 0, ef, scratch, size, worst, ID_MASK);

    for (;;) {
      // nearest not-yet-expanded list entry == candidate_set.top() (:268)
      int pos = -1;
#pragma unroll
      for (int e = 0; e < EPL; e++) {
        const unsigned m = __ballot_sync(FULL_MASK, !(L.v[e] & EXPANDED_BIT));  // empty slots have the bit set
        if (m && pos < 0) pos = e * 32 + __ffs(m) - 1;
      }
      if (pos < 0) break;
      const uint32_t node = L.val_at(pos);
#pragma unroll
      for (int e = 0; e < EPL; e++)
        if (e * 32 + lane == pos) L.v[e] |= EXPANDED_BIT;

      const uint8_t *rec = g.rec0 + (size_t)node * g.rec0_bytes;
      hops++;
      for (int c0 = 0; c0 < g.maxM0; c0 += 32) {
        const int j = c0 + lane;
        const uint32_t link = j < g.maxM0 ? __ldg(reinterpret_cast<const uint32_t *>(rec) + j) : EMPTY_LINK;
        const bool valid = link != EMPTY_LINK;
        float d = CUDART_INF_F;
        if (valid) d = score<CR, CB>(T, rec + g.code_off0 + (size_t)j * g.code_row, g.M, g.Ks);
        const int nv = __popc(__ballot_sync(FULL_MASK, valid));
        nbrs += nv;
        evals += nv;
        // admission test of :306 for the whole neighbour list at once; candidates that a sequential
        // scan would reject after lowerBound fell land beyond position ef-1 in the merge and drop out
        L.merge(d, link, valid && d < worst, ef, scratch, size, worst, ID_MASK);
        if (nv < 32) break;
      }
    }
    write_results<EPL>(g, p, q, L, lane, hops, nbrs, evals);
  }
}

// ---- v3: one neighbour chunk per node (maxM0 <= 32, the reference default M=16) ------------------
// Software-pipelined hop: as soon as the neighbours are scored the most likely next node is known
// (the nearest unexpanded list entry, or a new candidate that beats it), so its 384 B record is
// requested BEFORE the merge and the DRAM round trip overlaps the merge work.  The next node is then
// determined exactly from the merged list; a wrong guess only costs a reload.
template <int EPL, int CR, int CB, bool SMEM_TABLE>
__global__ void hnsw_walk_fast(const GraphDev g, const SearchParams p, const int table_stride_bytes) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int TS = g.M * g.Ks;
  constexpr int CAP = 32 * EPL;
  // [nwarps x table (SMEM_TABLE only)] [nwarps x (CAP list mirror + 32 candidate slots) uint2]
  float *Ts = reinterpret_cast<float *>(smem_raw + (size_t)warp * table_stride_bytes);
  // [nwarps x table] [nwarps x (CAP list mirror + 32 candidate slots + 1 mbarrier) x 8 B]
  uint2 *sl = reinterpret_cast<uint2 *>(smem_raw + (size_t)nwarps * table_stride_bytes) + (size_t)warp * (CAP + 33);
  uint2 *cbuf = sl + CAP;
  uint64_t *tbar = reinterpret_cast<uint64_t *>(cbuf + 32);
  const bool tma_table = SMEM_TABLE && ((TS * 4) % 16 == 0) && ((reinterpret_cast<uintptr_t>(p.tables) & 15) == 0);
  uint32_t tphase = 0;
  if (tma_table) {
    if (lane == 0) mbar_init(tbar, 1);
    __syncwarp();
  }
  const int ef = p.ef;
  const unsigned lt_mask = (1u << lane) - 1u;
  constexpr int CW = CR > 0 ? CR / 4 : 1;

  for (;;) {
    const int64_t q = next_query(p.work_counter, lane);
    if (q >= p.B) break;
    const float *T;
    if (SMEM_TABLE) {
      __syncwarp();  // every lane is done reading the previous query's table
      if (tma_table) {
        if (lane == 0) {
          mbar_expect_tx(tbar, (uint32_t)TS * 4u);
          bulk_g2s(Ts, p.tables + q * TS, (uint32_t)TS * 4u, tbar);
        }
        mbar_wait(tbar, tphase);
        tphase ^= 1u;
      } else {
        load_table(Ts, p.tables + q * TS, TS, lane);
        __syncwarp();
      }
      T = Ts;
    } else {
      T = p.tables + q * TS;
    }

    Walk w = descend<CR, CB>(g, T, lane);
    int hops = w.hops, nbrs = w.nbrs, evals = w.evals + 1;  // searchBaseLayerST re-scores the entry (:255)

    // list: registers (striped) + shared mirror; the entry node starts expanded (it is hop 0)
    WarpList<EPL> L;
    L.clear();
    // the shared mirror is padded with +inf keys so the rank search below needs no bounds
#pragma unroll
    for (int e = 0; e < EPL; e++) sl[e * 32 + lane] = make_uint2(0x7f800000u, LIST_EMPTY_VAL);
    __syncwarp();
    if (lane == 0) {
      L.k[0] = w.dist;
      L.v[0] = w.node | EXPANDED_BIT;
      sl[0] = make_uint2(__float_as_uint(w.dist), w.node | EXPANDED_BIT);
    }
    int size = 1;
    float worst = (ef == 1) ? w.dist : CUDART_INF_F;  // lowerBound (:306); +inf while the list is not full
    __syncwarp();

    // current record in registers
    uint32_t link;
    uint32_t cw[CW];
    const uint8_t *code_ptr = nullptr;
    const bool lane_has_slot = lane < g.maxM0;
    const uint8_t *lane_link_base = g.rec0 + 4 * lane;
    const uint8_t *lane_code_base = g.rec0 + g.code_off0 + (size_t)lane * g.code_row;
    const uint32_t rec_bytes = (uint32_t)g.rec0_bytes;
    auto load_record = [&](uint32_t node, uint32_t &lk, uint32_t *words, const uint8_t *&cptr) {
      const size_t off = (size_t)node * rec_bytes;
      lk = lane_has_slot ? __ldg(reinterpret_cast<const uint32_t *>(lane_link_base + off)) : EMPTY_LINK;
      cptr = lane_code_base + off;
      if (CR > 0 && lane_has_slot) {
        CodeWords<(CR > 0 ? CR : 4)> c;
        c.load(cptr);
#pragma unroll
        for (int i = 0; i < CW; i++) words[i] = c.w[i];
      }
    };
    load_record(w.node, link, cw, code_ptr);

    for (;;) {
      hops++;
      // ---- nearest unexpanded entry of the current list; request its record right away: unless this
      // hop finds something closer it is the next node, and its DRAM round trip then overlaps the
      // whole hop (scoring + merge) ----
      int pos2 = -1;
#pragma unroll
      for (int e = 0; e < EPL; e++) {
        const unsigned m = __ballot_sync(FULL_MASK, !(L.v[e] & EXPANDED_BIT));
        if (m && pos2 < 0) pos2 = e * 32 + __ffs(m) - 1;
      }
      uint2 e2 = make_uint2(0x7f800000u, LIST_EMPTY_VAL);
      if (pos2 >= 0) e2 = sl[pos2];
      uint32_t pred = LIST_EMPTY_VAL;
      uint32_t link_n = EMPTY_LINK;
      uint32_t cw_n[CW];
      const uint8_t *code_ptr_n = nullptr;
      if (pos2 >= 0) {
        pred = e2.y & ID_MASK;
        load_record(pred, link_n, cw_n, code_ptr_n);
      }
      // ---- score the neighbour list (one lane = one neighbour, m sequential) ----
      const bool valid = link != EMPTY_LINK;
      float d = CUDART_INF_F;
      if (valid) {
        if (CR > 0) {
          CodeWords<(CR > 0 ? CR : 4)> c;
#pragma unroll
          for (int i = 0; i < CW; i++) c.w[i] = cw[i];
          d = pq_lookup<(CR > 0 ? CR : 4), CB>(T, c, g.Ks);
        } else {
          d = pq_lookup_mem<CB>(T, code_ptr, g.M, g.Ks);
        }
      }
      const int nv = __popc(__ballot_sync(FULL_MASK, valid));
      nbrs += nv;
      evals += nv;

      // ---- admission (:306) for the whole list at once: rank by binary search, drop re-encounters ----
      const bool take = valid && d < worst;
      const unsigned offered = __ballot_sync(FULL_MASK, take);
      unsigned live = 0;
      int base = 0;
      if (offered) {
        bool dup = false;
        if (take) {
          // branch-free lower bound over the CAP-entry (inf padded) mirror; d < worst <= key[ef-1]
          // guarantees the count fits in [0, CAP-1]
          int lo = 0;
#pragma unroll
          for (int step = CAP / 2; step >= 1; step >>= 1) lo += (__uint_as_float(sl[lo + step - 1].x) <= d) ? step : 0;
          base = lo;  // number of list keys <= d: the candidate lands after its equals
          for (int t = base - 1; t >= 0; t--) {  // an id can only match where the key matches
            const uint2 x = sl[t];
            if (__uint_as_float(x.x) != d) break;
            if ((x.y & ID_MASK) == link) {
              dup = true;
              break;
            }
          }
        }
        live = __ballot_sync(FULL_MASK, take && !dup);
      }

      // ---- a new candidate beats the entry whose record is already on its way: re-aim the prefetch ----
      const unsigned fm = __ballot_sync(FULL_MASK, ((live >> lane) & 1u) && d < __uint_as_float(e2.x));
      if (fm) {
        pred = __shfl_sync(FULL_MASK, link, __ffs(fm) - 1);
        load_record(pred, link_n, cw_n, code_ptr_n);
      }

      // ---- merge the live candidates into the list ----
      int pos = pos2;
      if (live) {
        const int r = __popc(live & lt_mask);
        const bool mine = (live >> lane) & 1u;
        if (mine) cbuf[r] = make_uint2(__float_as_uint(d), link);
        __syncwarp();
        const int np_live = __popc(live);
        int shift[EPL];
#pragma unroll
        for (int e = 0; e < EPL; e++) shift[e] = 0;
        int crank = 0;
        for (int i = 0; i < np_live; i++) {
          const float dc = __uint_as_float(cbuf[i].x);
#pragma unroll
          for (int e = 0; e < EPL; e++) shift[e] += (dc < L.k[e]) ? 1 : 0;
          crank += ((dc < d) || (dc == d && i < r)) ? 1 : 0;
        }
#pragma unroll
        for (int e = 0; e < EPL; e++) {
          const int np = e * 32 + lane + shift[e];
          if (L.v[e] != LIST_EMPTY_VAL && np < ef) sl[np] = make_uint2(__float_as_uint(L.k[e]), L.v[e]);
        }
        if (mine) {
          const int np = base + crank;
          if (np < ef) sl[np] = make_uint2(__float_as_uint(d), link);
        }
        size = min(size + np_live, ef);
        __syncwarp();
#pragma unroll
        for (int e = 0; e < EPL; e++) {
          const int ps = e * 32 + lane;
          if (ps < size) {
            const uint2 t = sl[ps];
            L.k[e] = __uint_as_float(t.x);
            L.v[e] = t.y;
          } else {
            L.k[e] = CUDART_INF_F;
            L.v[e] = LIST_EMPTY_VAL;
          }
        }
        if (size == ef) worst = __uint_as_float(sl[ef - 1].x);
        // no live candidate beats the old nearest-unexpanded entry => it did not move and is still first
        if (fm || pos2 < 0) {
          pos = -1;
#pragma unroll
          for (int e = 0; e < EPL; e++) {
            const unsigned m = __ballot_sync(FULL_MASK, !(L.v[e] & EXPANDED_BIT));
            if (m && pos < 0) pos = e * 32 + __ffs(m) - 1;
          }
        }
      }
      if (pos < 0) break;  // candidate_set exhausted (:266)

      // ---- expand `pos`: flag it in both copies, take its record ----
      const uint32_t node = sl[pos].y & ID_MASK;
#pragma unroll
      for (int e = 0; e < EPL; e++)
        if (e * 32 + lane == pos) {
          L.v[e] |= EXPANDED_BIT;
          sl[pos].y = L.v[e];
        }
      __syncwarp();
      if (node == pred) {
        link = link_n;
        code_ptr = code_ptr_n;
#pragma unroll
        for (int i = 0; i < CW; i++) cw[i] = cw_n[i];
      } else {
        load_record(node, link, cw, code_ptr);
      }
    }
    write_results<EPL>(g, p, q, L, lane, hops, nbrs, evals);
  }
}

// =================================================================================================
// flagged path: deletions and/or filter WITHOUT a visited set or a candidate bag
// =================================================================================================
// Same single-list idea as hnsw_walk_fast, extended to nodes that are traversed but not admitted:
// every evaluated node that the reference would push to candidate_set (:306 / :413) is kept in ONE
// sorted list (capacity CAP = 32*EPL, chosen by the host from the filter's selectivity) with a PASS
// flag (admitted to top_candidates: passes the filter / is not deleted).  lowerBound is read off the
// list: the key of the ef-th passing entry once ef of them exist (everything behind it is dropped --
// those candidates have d >= lowerBound and are never expanded, :270 / :371), else the key of the last
// passing entry, else FLT_MAX -- exactly the values top_candidates.top() takes in the reference.
// While fewer than ef entries pass nothing is dropped, which is what makes the walk exact without a
// visited set: a re-encountered node is either still listed (id compare on equal keys) or was dropped
// with d >= a lowerBound that has only fallen since.  If the list would overflow its capacity the
// query is flagged (found = -1) and the host re-runs the batch on the bitmap kernel below.
constexpr uint32_t PASS_BIT = 0x40000000u;
constexpr uint32_t ID_MASK30 = 0x3fffffffu;

// PQF: query q is admitted by its own bitmap p.query_filter[q] (nullptr = "not deleted"), chosen per query
template <int EPL, int CR, int CB, bool PQF>
__global__ void hnsw_walk_flagged(const GraphDev g, const SearchParams p, const int has_del, const int table_stride_bytes) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int TS = g.M * g.Ks;
  constexpr int CAP = 32 * EPL;
  float *Ts = reinterpret_cast<float *>(smem_raw + (size_t)warp * table_stride_bytes);
  uint2 *sl = reinterpret_cast<uint2 *>(smem_raw + (size_t)nwarps * table_stride_bytes) + (size_t)warp * (CAP + 33);
  uint2 *cbuf = sl + CAP;
  uint64_t *tbar = reinterpret_cast<uint64_t *>(cbuf + 32);
  const bool tma_table = ((TS * 4) % 16 == 0) && ((reinterpret_cast<uintptr_t>(p.tables) & 15) == 0);
  uint32_t tphase = 0;
  if (tma_table) {
    if (lane == 0) mbar_init(tbar, 1);
    __syncwarp();
  }
  const int ef = p.ef;
  const int k = p.k;
  const unsigned lt_mask = (1u << lane) - 1u;
  const unsigned le_mask = lt_mask | (1u << lane);
  constexpr int CW = CR / 4;
  const uint32_t *filter = p.filter;
  bool use_filter = filter != nullptr;
  const uint32_t *delbits = g.deleted;
  auto passes = [&](uint32_t id) -> bool {
    if (use_filter) return (__ldg(filter + (id >> 5)) >> (id & 31)) & 1u;   // :353-354, :423-426
    return !((__ldg(delbits + (id >> 5)) >> (id & 31)) & 1u);              // :254, :314
  };
  const float FLT_MAX_ = 3.402823466e+38f;

  for (;;) {
    const int64_t q = next_query(p.work_counter, lane);
    if (q >= p.B) break;
    if constexpr (PQF) {
      filter = p.query_filter[q];
      use_filter = filter != nullptr;
    }
    __syncwarp();
    if (tma_table) {
      if (lane == 0) {
        mbar_expect_tx(tbar, (uint32_t)TS * 4u);
        bulk_g2s(Ts, p.tables + q * TS, (uint32_t)TS * 4u, tbar);
      }
      mbar_wait(tbar, tphase);
      tphase ^= 1u;
    } else {
      load_table(Ts, p.tables + q * TS, TS, lane);
      __syncwarp();
    }
    const float *T = Ts;

    Walk w = descend<CR, CB>(g, T, lane);
    int hops = w.hops, nbrs = w.nbrs, evals = w.evals + 1;

    WarpList<EPL> L;
    L.clear();
#pragma unroll
    for (int e = 0; e < EPL; e++) sl[e * 32 + lane] = make_uint2(0x7f800000u, LIST_EMPTY_VAL);
    __syncwarp();
    const bool ep_pass = passes(w.node);
    const uint32_t ep_val = w.node | EXPANDED_BIT | (ep_pass ? PASS_BIT : 0u);
    if (lane == 0) {
      L.k[0] = w.dist;
      L.v[0] = ep_val;
      sl[0] = make_uint2(__float_as_uint(w.dist), ep_val);
    }
    int size = 1, npass = ep_pass ? 1 : 0;
    float lb = ep_pass ? w.dist : FLT_MAX_;   // lowerBound of the reference (:256 / :260)
    bool aborted = false;
    __syncwarp();

    uint32_t link;
    uint32_t cw[CW];
    const bool lane_has_slot = lane < g.maxM0;
    const uint8_t *lane_link_base = g.rec0 + 4 * lane;
    const uint8_t *lane_code_base = g.rec0 + g.code_off0 + (size_t)lane * g.code_row;
    const uint32_t rec_bytes = (uint32_t)g.rec0_bytes;
    auto load_record = [&](uint32_t node, uint32_t &lk, uint32_t *words) {
      const size_t off = (size_t)node * rec_bytes;
      lk = lane_has_slot ? __ldg(reinterpret_cast<const uint32_t *>(lane_link_base + off)) : EMPTY_LINK;
      if (lane_has_slot) {
        CodeWords<CR> c;
        c.load(lane_code_base + off);
#pragma unroll
        for (int i = 0; i < CW; i++) words[i] = c.w[i];
      }
    };
    load_record(w.node, link, cw);

    for (;;) {
      hops++;
      int pos2 = -1;
#pragma unroll
      for (int e = 0; e < EPL; e++) {
        const unsigned m = __ballot_sync(FULL_MASK, !(L.v[e] & EXPANDED_BIT));
        if (m && pos2 < 0) pos2 = e * 32 + __ffs(m) - 1;
      }
      uint2 e2 = make_uint2(0x7f800000u, LIST_EMPTY_VAL);
      if (pos2 >= 0) e2 = sl[pos2];
      uint32_t pred = LIST_EMPTY_VAL;
      uint32_t link_n = EMPTY_LINK;
      uint32_t cw_n[CW];
      if (pos2 >= 0) {  // the likely next node: its record travels while this hop is scored and merged
        pred = e2.y & ID_MASK30;
        load_record(pred, link_n, cw_n);
      }
      const bool valid = link != EMPTY_LINK;
      float d = CUDART_INF_F;
      bool pf = false;
      if (valid) {
        pf = passes(link);
        CodeWords<CR> c;
#pragma unroll
        for (int i = 0; i < CW; i++) c.w[i] = cw[i];
        d = pq_lookup<CR, CB>(T, c, g.Ks);
      }
      const int nv = __popc(__ballot_sync(FULL_MASK, valid));
      nbrs += nv;
      evals += nv;

      // admission to candidate_set: top_candidates.size() < ef || lowerBound > dist (:306 / :413)
      const bool take = valid && (npass < ef || d < lb);
      const unsigned offered = __ballot_sync(FULL_MASK, take);
      unsigned live = 0;
      int base = 0;
      if (offered) {
        bool dup = false;
        if (take) {
          int lo = 0;
#pragma unroll
          for (int step = CAP / 2; step >= 1; step >>= 1) lo += (__uint_as_float(sl[lo + step - 1].x) <= d) ? step : 0;
          base = lo;
          for (int t = base - 1; t >= 0; t--) {
            const uint2 x = sl[t];
            if (__uint_as_float(x.x) != d) break;
            if ((x.y & ID_MASK30) == link) {
              dup = true;
              break;
            }
          }
        }
        live = __ballot_sync(FULL_MASK, take && !dup);
      }
      const int np_live = __popc(live);
      if (size + np_live > CAP) {  // capacity chosen by the host was too small for this query
        aborted = true;
        break;
      }

      const unsigned fm = __ballot_sync(FULL_MASK, ((live >> lane) & 1u) && d < __uint_as_float(e2.x));
      if (fm) {
        pred = __shfl_sync(FULL_MASK, link, __ffs(fm) - 1);
        load_record(pred, link_n, cw_n);
      }

      int pos = pos2;
      if (live) {
        const int r = __popc(live & lt_mask);
        const bool mine = (live >> lane) & 1u;
        const uint32_t myval = link | (pf ? PASS_BIT : 0u);
        if (mine) cbuf[r] = make_uint2(__float_as_uint(d), myval);
        __syncwarp();
        int shift[EPL];
#pragma unroll
        for (int e = 0; e < EPL; e++) shift[e] = 0;
        int crank = 0;
        for (int i = 0; i < np_live; i++) {
          const float dc = __uint_as_float(cbuf[i].x);
#pragma unroll
          for (int e = 0; e < EPL; e++) shift[e] += (dc < L.k[e]) ? 1 : 0;
          crank += ((dc < d) || (dc == d && i < r)) ? 1 : 0;
        }
#pragma unroll
        for (int e = 0; e < EPL; e++) {
          const int np = e * 32 + lane + shift[e];
          if (L.v[e] != LIST_EMPTY_VAL) sl[np] = make_uint2(__float_as_uint(L.k[e]), L.v[e]);
        }
        if (mine) sl[base + crank] = make_uint2(__float_as_uint(d), myval);
        const int merged = size + np_live;
        __syncwarp();
#pragma unroll
        for (int e = 0; e < EPL; e++) {
          const int ps = e * 32 + lane;
          if (ps < merged) {
            const uint2 t = sl[ps];
            L.k[e] = __uint_as_float(t.x);
            L.v[e] = t.y;
          } else {
            L.k[e] = CUDART_INF_F;
            L.v[e] = LIST_EMPTY_VAL;
          }
        }
        // ---- lowerBound = top_candidates.top() (:320-321) read off the list; drop what lies beyond it ----
        unsigned pm[EPL];
        int total = 0;
#pragma unroll
        for (int e = 0; e < EPL; e++) {
          pm[e] = __ballot_sync(FULL_MASK, L.v[e] != LIST_EMPTY_VAL && (L.v[e] & PASS_BIT));
          total += __popc(pm[e]);
        }
        size = merged;
        if (total >= ef) {
          int cum = 0, P = -1;
#pragma unroll
          for (int e = 0; e < EPL; e++) {
            const int c = __popc(pm[e]);
            if (P < 0 && cum + c >= ef) {
              const int need = ef - cum;
              const unsigned hit = __ballot_sync(FULL_MASK, ((pm[e] >> lane) & 1u) && __popc(pm[e] & le_mask) == need);
              P = e * 32 + __ffs(hit) - 1;
            }
            cum += c;
          }
          const int newsize = P + 1;
#pragma unroll
          for (int e = 0; e < EPL; e++) {
            const int ps = e * 32 + lane;
            if (ps >= newsize && ps < merged) {
              L.k[e] = CUDART_INF_F;
              L.v[e] = LIST_EMPTY_VAL;
              sl[ps] = make_uint2(0x7f800000u, LIST_EMPTY_VAL);
            }
          }
          size = newsize;
          npass = ef;
          lb = __uint_as_float(sl[P].x);
        } else {
          npass = total;
          if (total > 0) {
            int plast = -1;
#pragma unroll
            for (int e = EPL - 1; e >= 0; e--)
              if (plast < 0 && pm[e]) plast = e * 32 + 31 - __clz(pm[e]);
            lb = __uint_as_float(sl[plast].x);
          }
        }
        __syncwarp();
        pos = -1;
#pragma unroll
        for (int e = 0; e < EPL; e++) {
          const unsigned m = __ballot_sync(FULL_MASK, !(L.v[e] & EXPANDED_BIT));
          if (m && pos < 0) pos = e * 32 + __ffs(m) - 1;
        }
      }
      if (pos < 0) break;
      const uint2 nx = sl[pos];
      const float nkey = __uint_as_float(nx.x);
      if (use_filter) {
        if (nkey > lb) break;                                                      // :371
      } else if (nkey > lb && (npass == ef || !has_del)) {
        break;                                                                     // :270
      }
      const uint32_t node = nx.y & ID_MASK30;
#pragma unroll
      for (int e = 0; e < EPL; e++)
        if (e * 32 + lane == pos) {
          L.v[e] |= EXPANDED_BIT;
          sl[pos].y = L.v[e];
        }
      __syncwarp();
      if (node == pred) {
        link = link_n;
#pragma unroll
        for (int i = 0; i < CW; i++) cw[i] = cw_n[i];
      } else {
        load_record(node, link, cw);
      }
    }

    // ---- results: the first k passing entries, ascending (dist, label) ----
    if (aborted) {
      if (lane == 0) p.out_found[q] = -1;
      continue;
    }
    int cum = 0;
    bool tie = false;
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const bool pass = L.v[e] != LIST_EMPTY_VAL && (L.v[e] & PASS_BIT);
      const unsigned m = __ballot_sync(FULL_MASK, pass);
      const int r = cum + __popc(m & lt_mask);
      if (pass && r < k) {
        p.out_dists[q * k + r] = L.k[e];
        p.out_labels[q * k + r] = __ldg(g.labels + (L.v[e] & ID_MASK30));
      }
      float nk = __shfl_down_sync(FULL_MASK, L.k[e], 1);
      const float first_next = (e + 1 < EPL) ? __shfl_sync(FULL_MASK, L.k[(e + 1 < EPL) ? e + 1 : e], 0) : CUDART_INF_F;
      if (lane == 31) nk = first_next;
      tie |= (L.v[e] != LIST_EMPTY_VAL) && (nk == L.k[e]);
      cum += __popc(m);
    }
    const int found = min(cum, k);
    for (int r = found + lane; r < k; r += 32) {
      p.out_dists[q * k + r] = CUDART_INF_F;
      p.out_labels[q * k + r] = (uint64_t)UINT64_MAX;
    }
    if (__any_sync(FULL_MASK, tie)) {
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
}

// =================================================================================================
// bitmap path: deletions and/or filter (literal two-structure walk with an exact visited set)
// =================================================================================================
// PQF: as in hnsw_walk_flagged, the bitmap of query row q is p.query_filter[q]
template <int EPL, int CR, int CB, bool SMEM_TABLE, bool PQF>
__global__ void hnsw_walk_general(const GraphDev g, const SearchParams p, const int has_del, const int table_stride_bytes) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int TS = g.M * g.Ks;
  float *Ts = reinterpret_cast<float *>(smem_raw + (size_t)warp * table_stride_bytes);
  // [nwarps x table] [nwarps x (32*EPL merge scratch + SBAG bag) x 8 B]
  uint2 *scratch = reinterpret_cast<uint2 *>(smem_raw + (size_t)nwarps * table_stride_bytes) + (size_t)warp * (32 * EPL + SBAG);
  uint64_t *sbag = reinterpret_cast<uint64_t *>(scratch + 32 * EPL);
  const unsigned lt_mask = (1u << lane) - 1u;
  const int ef = p.ef;
  const int64_t slot = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  uint32_t *vis = p.visited + slot * p.visited_words;
  uint32_t *touched = p.touched + slot * (int64_t)p.touched_cap;
  uint64_t *gbag = p.cand + slot * (int64_t)p.cand_cap;
  const uint32_t *filter = p.filter;
  bool use_filter = filter != nullptr;

  for (;;) {
    const int64_t wi = next_query(p.work_counter, lane);
    if (wi >= p.B) break;
    const int64_t q = p.qmap ? (int64_t)__ldg(p.qmap + wi) : wi;  // subset re-run: outputs stay indexed by query row
    if constexpr (PQF) {
      filter = p.query_filter[q];
      use_filter = filter != nullptr;
    }
    const float *T;
    if (SMEM_TABLE) {
      __syncwarp();
      load_table(Ts, p.tables + q * TS, TS, lane);
      __syncwarp();
      T = Ts;
    } else {
      T = p.tables + q * TS;
    }

    Walk w = descend<CR, CB>(g, T, lane);
    int hops = w.hops, nbrs = w.nbrs, evals = w.evals;

    WarpList<EPL> L;  // top_candidates: admitted entries only
    L.clear();
    // candidate_set: an unordered bag, first SBAG entries in shared memory, the rest in global scratch
    int topsize = 0, ns = 0, ng = 0, ntouched = 0;
    bool overflow = false;
    float lower;
    {
      const uint32_t ep = w.node;
      bool ok;
      if (use_filter) ok = (filter[ep >> 5] >> (ep & 31)) & 1u;                    // :353-354
      else ok = !has_del || !((g.deleted[ep >> 5] >> (ep & 31)) & 1u);             // :254
      if (ok) {
        evals++;
        lower = w.dist;
        L.insert(w.dist, ep, ef);
        topsize = 1;
        if (lane == 0) sbag[0] = pack_cand(w.dist, ep);
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
        float od = __shfl_xor_sync(FULL_MASK, bd, o);
        int oi = __shfl_xor_sync(FULL_MASK, bi, o);
        uint32_t oid = __shfl_xor_sync(FULL_MASK, bid, o);
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
      // request the record now; the bag maintenance below overlaps the DRAM round trip
      const uint8_t *rec = g.rec0 + (size_t)bid * g.rec0_bytes;
      uint32_t link0 = (lane < g.maxM0) ? __ldg(reinterpret_cast<const uint32_t *>(rec) + lane) : EMPTY_LINK;
      // pop: move the last entry of that part into the hole
      if (lane == 0) {
        if (bi < SBAG) sbag[bi] = sbag[ns - 1];
        else gbag[bi - SBAG] = gbag[ng - 1];
      }
      if (bi < SBAG) ns--;
      else ng--;
      __syncwarp();
      // candidates beyond lowerBound are dead once top is full (lowerBound only falls): drop them now and
      // then so the nearest-candidate scan stays short and the shared part does not spill
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
        const uint32_t link = (c0 == 0) ? link0 : (j < g.maxM0 ? __ldg(reinterpret_cast<const uint32_t *>(rec) + j) : EMPTY_LINK);
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
          d = score<CR, CB>(T, rec + g.code_off0 + (size_t)j * g.code_row, g.M, g.Ks);
          if (use_filter) admit = (filter[link >> 5] >> (link & 31)) & 1u;        // :423-426
          else admit = !has_del || !((g.deleted[link >> 5] >> (link & 31)) & 1u);  // :314
        }
        // Admission (:306 / :413) for the whole neighbour list at once.  lowerBound only falls once top
        // is full, so testing against its value at the start of the list admits a superset of what the
        // sequential scan admits; the extras have d >= the final lowerBound, are never expanded (the
        // loop breaks first, :270 / :371) and fall off the top list in the merge -- same results.
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
      if (ntouched > p.touched_cap) {  // log overflowed: wipe everything
        for (int64_t i = lane; i < p.visited_words; i += 32) vis[i] = 0u;
      }
    }
    if (overflow && lane == 0) atomicExch(p.overflow_flag, 1);
    __syncwarp();
    write_results<EPL>(g, p, q, L, lane, hops, nbrs, evals);
  }
}

// label list -> bitmap by internal id.  labels of the index are unique; the allowed list is
// first marked in a bitmap over label values, then gathered by internal id.
__global__ void mark_labels_kernel(const uint64_t *__restrict__ allowed, int64_t n, uint32_t *__restrict__ by_label,
                                   uint64_t max_label) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t l = allowed[i];
  if (l <= max_label) atomicOr(by_label + (l >> 5), 1u << (l & 31));
}
__global__ void gather_filter_kernel(const uint64_t *__restrict__ labels, int64_t n, const uint32_t *__restrict__ by_label,
                                     uint32_t *__restrict__ by_id) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  if (i < n) {
    uint64_t l = labels[i];
    ok = (by_label[l >> 5] >> (l & 31)) & 1u;
  }
  unsigned m = __ballot_sync(FULL_MASK, ok);
  if ((threadIdx.x & 31) == 0 && (i < n)) by_id[i >> 5] = m;
}

// the reference layout's element size (4 + 4*maxM0 + code_row + 8) is not a multiple of 4 for odd
// code rows, so its fields are read bytewise
__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t *p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// level-0 walk records from the reference-layout records: [links | neighbour codes]
__global__ void pack_rec0_kernel(const uint8_t *__restrict__ raw, int64_t n, int size_per_elem, int offset_data,
                                 int maxM0, int code_row, int code_off0, int rec0_bytes, uint8_t *__restrict__ rec0) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t node = t / maxM0;
  const int j = (int)(t - node * maxM0);
  if (node >= n) return;
  const uint8_t *src = raw + node * size_per_elem;
  const unsigned cnt = (unsigned)src[0] | ((unsigned)src[1] << 8);
  uint8_t *dst = rec0 + node * rec0_bytes;
  uint32_t link = EMPTY_LINK;
  if ((unsigned)j < cnt) link = ld_u32_unaligned(src + 4 + 4 * j);
  *reinterpret_cast<uint32_t *>(dst + 4 * j) = link;
  uint8_t *cdst = dst + code_off0 + (size_t)j * code_row;
  if (link != EMPTY_LINK) {
    const uint8_t *csrc = raw + (size_t)link * size_per_elem + offset_data;
    for (int b = 0; b < code_row; b++) cdst[b] = csrc[b];
  } else {
    for (int b = 0; b < code_row; b++) cdst[b] = 0;
  }
}

struct LaunchGeom {
  int warps, ctas_per_sm, smem_bytes;
  bool smem_table;
};

LaunchGeom pick_geometry(annb_index *h, size_t table_bytes_in, size_t extra_per_warp, int max_warps) {
  const size_t table_bytes = (table_bytes_in + 15) / 16 * 16 + extra_per_warp;
  int optin = 0, per_sm = 0;
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device);
  cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, h->device);
  LaunchGeom best{4, 1, 0, false};
  if (table_bytes > (size_t)optin) {  // table does not fit: read it through L1/L2
    best.warps = std::min(8, max_warps);
    best.ctas_per_sm = 4;
    best.smem_bytes = (int)(best.warps * extra_per_warp);
    return best;
  }
  int best_total = 0;
  for (int W = 1; W <= max_warps; W++) {
    size_t need = W * table_bytes;
    if (need > (size_t)optin) break;
    int ctas = (int)((size_t)per_sm / (need + 1024));
    if (ctas < 1) continue;
    ctas = std::min(ctas, 32);
    int total = std::min(W * ctas, 32);  // beyond ~32 warps/SM the register file limits residency anyway
    if (total > best_total) {
      best_total = total;
      best.warps = W;
      best.ctas_per_sm = std::min(ctas, (32 + W - 1) / W);
      best.smem_bytes = (int)need;
      best.smem_table = true;
    }
  }
  if (h->opt_warps_per_cta > 0 && h->opt_warps_per_cta <= max_warps && h->opt_warps_per_cta * table_bytes <= (size_t)optin) {
    best.warps = (int)h->opt_warps_per_cta;
    best.smem_bytes = (int)(best.warps * table_bytes);
    best.ctas_per_sm = std::max(1, (int)((size_t)per_sm / (best.smem_bytes + 1024)));
    best.smem_table = true;
  }
  if (h->opt_ctas_per_sm > 0) best.ctas_per_sm = (int)h->opt_ctas_per_sm;
  return best;
}

// Sets the dynamic shared memory limit of `kern` for `geo` and asks how many of its CTAs fit on an SM.  Large EPL
// instantiations need > 64 registers/thread, so a CTA of 32 warps may not fit the register file: while none fits, the
// geometry is re-picked with half the warps.  *occ = resident CTAs per SM (at most geo.ctas_per_sm), 0 = none fits.
int fit_geometry(annb_index *h, const void *kern, size_t table_bytes, size_t extra, LaunchGeom &geo, int *occ) {
  for (int max_warps = 32;;) {
    if (geo.smem_bytes > 48 * 1024) ANNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, geo.smem_bytes));
    ANNB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, kern, geo.warps * 32, geo.smem_bytes));
    if (*occ >= 1 || max_warps == 1) break;
    max_warps = std::max(1, std::min(max_warps, geo.warps) / 2);
    geo = pick_geometry(h, table_bytes, extra, max_warps);
  }
  *occ = std::min(*occ, geo.ctas_per_sm);
  return ANNB_OK;
}

template <int EPL, int CR, int CB, bool SMEM_TABLE, bool PQF>
int launch_walk_t(annb_index *h, SearchParams &p, bool general, size_t table_bytes, size_t extra, LaunchGeom geo) {
  auto fast = h->gd.maxM0 > 32 ? hnsw_walk_chunked<EPL, CR, CB, SMEM_TABLE> : hnsw_walk_fast<EPL, CR, CB, SMEM_TABLE>;
  auto bitmap = hnsw_walk_general<EPL, CR, CB, SMEM_TABLE, PQF>;
  int occ;
  ANNB_TRY_RC(fit_geometry(h, general ? (const void *)bitmap : (const void *)fast, table_bytes, extra, geo, &occ));
  if (!occ) ANNB_FAIL(ANNB_ELIMIT, "kernel does not fit on this device (registers/shared memory)");
  const int table_stride = SMEM_TABLE ? (int)((table_bytes + 15) / 16 * 16) : 0;
  const int threads = geo.warps * 32;
  const int blocks = (int)std::min<int64_t>((int64_t)h->sm_count * occ, (p.B + geo.warps - 1) / geo.warps);
  ANNB_TRY_RC(walk_counter(h, p));
  if (general) {
    const int has_del = h->g.num_deleted > 0;
    return run_bitmap_walk(h, p, blocks, geo.warps, "general", [&](int b, const SearchParams &pr) {
      bitmap<<<b, threads, geo.smem_bytes, h->stream>>>(h->gd, pr, has_del, table_stride);
    });
  }
  fast<<<blocks, threads, geo.smem_bytes, h->stream>>>(h->gd, p, table_stride);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

template <int EPL, int CR, int CB, bool PQF>
int launch_walk(annb_index *h, const SearchParams &p_in, bool general) {
  SearchParams p = p_in;
  const size_t table_bytes = (size_t)h->M * h->Ks * sizeof(float);
  const size_t extra = (size_t)(32 * EPL + (general ? SBAG : (h->gd.maxM0 > 32 ? 0 : 33))) * sizeof(uint2);
  const LaunchGeom geo = pick_geometry(h, table_bytes, extra, 32);
  if (geo.smem_table) return launch_walk_t<EPL, CR, CB, true, PQF>(h, p, general, table_bytes, extra, geo);
  // One-byte codes have no global-table form: a row has at most 128 bytes (wider rows take hnsw_walk_wide), so the
  // table has at most 128 KB and, with at most 6 KB of list and bag, always fits the 227 KB of opt-in shared memory.
  if constexpr (CB == 1) ANNB_FAIL(ANNB_ESTATE, "internal: a one-byte-code walk table that does not fit in shared memory");
  else return launch_walk_t<EPL, CR, CB, false, PQF>(h, p, general, table_bytes, extra, geo);
}

// f(CR, CB) as std::integral_constant for the index's code rows: CR bytes per row held in registers, 0 = read from memory
template <typename F>
int with_code_row(const annb_index *h, F f) {
  using std::integral_constant;
  if (h->code_bytes == 1) {
    switch (h->gd.code_row) {
      case 4: return f(integral_constant<int, 4>(), integral_constant<int, 1>());
      case 8: return f(integral_constant<int, 8>(), integral_constant<int, 1>());
      case 16: return f(integral_constant<int, 16>(), integral_constant<int, 1>());
      case 32: return f(integral_constant<int, 32>(), integral_constant<int, 1>());
      default: return f(integral_constant<int, 0>(), integral_constant<int, 1>());
    }
  }
  switch (h->gd.code_row) {
    case 8: return f(integral_constant<int, 8>(), integral_constant<int, 2>());
    case 16: return f(integral_constant<int, 16>(), integral_constant<int, 2>());
    default: return f(integral_constant<int, 0>(), integral_constant<int, 2>());
  }
}

// ---- flagged walk launcher ---------------------------------------------------------------------------
template <int EPL, int CR, int CB>
int launch_flagged(annb_index *h, const SearchParams &p_in) {
  SearchParams p = p_in;
  const size_t table_bytes = (size_t)h->M * h->Ks * sizeof(float);
  const size_t extra = (size_t)(32 * EPL + 33) * sizeof(uint2);
  // not applicable (1): the caller falls back to the bitmap walk.  smem_table depends on the table size only, so
  // fit_geometry's smaller geometries keep it.
  LaunchGeom geo = pick_geometry(h, table_bytes, extra, 32);
  if (!geo.smem_table) return 1;
  auto kern = p.query_filter ? hnsw_walk_flagged<EPL, CR, CB, true> : hnsw_walk_flagged<EPL, CR, CB, false>;
  int occ;
  ANNB_TRY_RC(fit_geometry(h, (const void *)kern, table_bytes, extra, geo, &occ));
  if (!occ) return 1;
  ANNB_TRY_RC(walk_counter(h, p));
  const int blocks = (int)std::min<int64_t>((int64_t)h->sm_count * occ, (p.B + geo.warps - 1) / geo.warps);
  kern<<<blocks, geo.warps * 32, geo.smem_bytes, h->stream>>>(h->gd, p, h->g.num_deleted > 0 ? 1 : 0,
                                                             (int)((table_bytes + 15) / 16 * 16));
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

}  // namespace

int launch_search(annb_index *h, const SearchParams &p, int mode) {
  if (p.B == 0) return ANNB_OK;
  if (p.B >= (int64_t)0xffffffffll) ANNB_FAIL(ANNB_ELIMIT, "at most 2^32-2 queries per call");
  if (wide_rows(h)) return launch_walk_wide(h, p);  // every mode: the literal walk, table-free (walk_wide.cu)
  if (mode == 1) {  // filter and/or deletions: two register lists in hnsw_walk4's mapping where that applies (walk_flagged4.cu)
    const int rc = launch_walk4f(h, p);
    if (rc != 1) return rc;
    if (!p.tables) ANNB_FAIL(ANNB_ESTATE, "internal: no tables for the flagged walk");
  }
  if (mode == 1 && h->gd.maxM0 <= 32 && h->gd.n < (1ll << 30)) {
    // list capacity the flagged walk needs: every candidate down to the ef-th admitted one stays listed
    const double s = std::min(1.0, std::max(1e-4, (double)p.selectivity));
    // until the ef-th admitted node is found the list holds every evaluated node: about ef/s of them
    // (binomial spread ~ sqrt(ef/s)); 1.3x + 48 leaves > 4 sigma of head-room at the usual sizes
    const double need = (double)p.ef / s * 1.3 + 48.0;
    int epl = 0;
    for (int e : {2, 4, 8, 16})
      if (epl == 0 && e * 32 >= need && e * 32 >= p.ef) epl = e;
    if (h->opt_flagged_epl > 0 && h->opt_flagged_epl * 32 >= p.ef) epl = (int)h->opt_flagged_epl;
    auto flagged = [&](auto epl_c) {
      return with_code_row(h, [&](auto cr, auto cb) {
        if constexpr (decltype(cr)::value == 0) return 1;  // no register form of the row: not applicable
        else return launch_flagged<decltype(epl_c)::value, decltype(cr)::value, decltype(cb)::value>(h, p);
      });
    };
    int rc = 1;
    if (epl == 2 || epl == 4 || epl == 8 || epl == 16) rc = with_epl(32 * epl, flagged);
    if (rc != 1) return rc;  // launched (or failed for real); 1 = not applicable -> bitmap walk
  }
  const bool general = mode != 0;
  if (!general && walk4_applicable(h)) {  // the plain search: K1 fused into the walk (walk_fused.cu)
    const int rc = launch_walk4(h, p);
    if (rc != 1) return rc;
  }
  if (!p.tables) ANNB_FAIL(ANNB_ESTATE, "internal: no tables for the walk");
  return with_epl(p.ef, [&](auto epl) {
    return with_code_row(h, [&](auto cr, auto cb) {
      constexpr int EPL = decltype(epl)::value, CR = decltype(cr)::value, CB = decltype(cb)::value;
      if (general && p.query_filter) return launch_walk<EPL, CR, CB, true>(h, p, general);
      return launch_walk<EPL, CR, CB, false>(h, p, general);
    });
  });
}

int search_route(const annb_index *h, int ef, bool filtered, double selectivity, bool *fuse, bool *walk4f) {
  const bool general = filtered || h->g.num_deleted > 0 || h->opt_force_general;
  const int mode = !general ? 0 : (h->opt_force_general == 2 ? 2 : 1);
  const bool w4f = mode == 1 && walk4f_applicable(h, ef, selectivity);
  // launch_search builds no tables: a walk without them must be one that builds its own (hnsw_walk_wide always does)
  if (fuse) *fuse = wide_rows(h) || (walk4_can_fuse(h) && (mode == 0 || w4f));
  if (walk4f) *walk4f = w4f;
  return mode;
}

double search_selectivity(const annb_index *h, bool filtered, int64_t count) {
  const double n = (double)std::max<int64_t>(1, h->gd.n);
  return filtered ? std::min<double>(1.0, (double)count / n) : 1.0 - (double)h->g.num_deleted / n;
}

int walk_counter(annb_index *h, SearchParams &p) {
  if (!p.work_counter) ANNB_TRY_RC(annb_scratch(h, 4, 256, (void **)&p.work_counter));
  ANNB_CUDA(cudaMemsetAsync(p.work_counter, 0, 8, h->stream));
  p.overflow_flag = reinterpret_cast<int32_t *>(p.work_counter + 1);
  return ANNB_OK;
}

int launch_pack_rec0(annb_index *h, const uint8_t *d_level0_raw, int64_t n) {
  if (n == 0) return ANNB_OK;
  const int64_t total = n * h->gd.maxM0;
  const int code_row = wide_rows(h) ? 0 : h->gd.code_row;  // wide rows: links-only records
  pack_rec0_kernel<<<(unsigned)((total + 255) / 256), 256, 0, h->stream>>>(
      d_level0_raw, n, (int)h->g.size_per_elem, (int)h->g.offset_data, h->gd.maxM0, code_row, h->gd.code_off0,
      h->gd.rec0_bytes,
      h->d_rec0);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

// patch of the device graph: staged[i] (one packed record) -> dst[ids[i]]
__global__ void scatter_records_kernel(const uint8_t *__restrict__ staged, const uint32_t *__restrict__ ids, int64_t cnt, int words,
                                       uint8_t *__restrict__ dst) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t i = t / words;
  if (i >= cnt) return;
  const int w = (int)(t - i * words);
  reinterpret_cast<uint32_t *>(dst + (size_t)ids[i] * words * 4)[w] = reinterpret_cast<const uint32_t *>(staged + (size_t)i * words * 4)[w];
}

int launch_scatter_records(annb_index *h, const uint8_t *d_staged, const uint32_t *d_ids, int64_t cnt, int rec_bytes, uint8_t *d_dst) {
  if (cnt == 0) return ANNB_OK;
  const int words = rec_bytes / 4;
  const int64_t total = cnt * words;
  scatter_records_kernel<<<(unsigned)((total + 255) / 256), 256, 0, h->stream>>>(d_staged, d_ids, cnt, words, d_dst);
  h->launches++;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}

int launch_filter_bitmap(annb_index *h, const uint64_t *d_filter_labels, int64_t n_filter, uint32_t *d_by_label,
                         uint32_t *d_by_id) {
  const int64_t n = h->gd.n;
  const size_t words = (size_t)(h->max_label >> 5) + 1;
  ANNB_CUDA(cudaMemsetAsync(d_by_label, 0, words * 4, h->stream));
  if (n_filter > 0)
    mark_labels_kernel<<<(unsigned)((n_filter + 255) / 256), 256, 0, h->stream>>>(d_filter_labels, n_filter, d_by_label,
                                                                               h->max_label);
  const int64_t padded = (n + 31) / 32 * 32;
  if (n > 0)  // an empty graph has no row to gather (and a launch of 0 blocks is an error)
    gather_filter_kernel<<<(unsigned)((padded + 255) / 256), 256, 0, h->stream>>>(h->d_labels, n, d_by_label, d_by_id);
  h->launches += 2;
  ANNB_CUDA(cudaGetLastError());
  return ANNB_OK;
}
