// walk_fused.cu -- K1+K3 in one kernel: the warp that walks a query first builds that query's ADC table
// straight into its own shared-memory slot, then runs the HNSW walk over PQ codes out of registers.
//
// Reference semantics (unchanged from hnsw_search.cu, where the equivalence argument lives):
//   table : batch_precompute_adc_table[_ip]  bindings/pq_bindings.pyx:149-274 (+ pq.py:316-322 epilogue)
//           T[m][c] = sum_j (cb[m][c][j] - q[m*ds+j])^2, j sequential, sub / mul / add rounded separately
//   walk  : searchKnn  include/hnswlib/hnswalg.h:1237-1295 = greedy descent (:1248-1274) +
//           searchBaseLayerST (:243-329) with PQLookup (include/hnswlib/space_pq.h:16-37)
//
// What is different from hnsw_walk_fast (round 1), and why -- that kernel was issue-bound at ~305 warp
// instructions per hop:
//   * compile-time M and Ks = 256, u8 codes: a table lookup is byte-extract + LDS with an immediate
//     row offset + FADD; no run-time m*Ks+code / node*rec_bytes integer chains.
//   * the ef-bounded result list lives ONLY in registers, blocked (lane l holds positions l*EPL..),
//     keys as order-preserving u32 images of the fp32 distances so that warp minima are one REDUX.
//     No shared-memory mirror, no binary search, no rank loops, no __syncwarp in the hop.
//   * candidates of a hop are consumed smallest-first: the first one that is not already listed is, if
//     it beats the nearest unexpanded list entry, exactly the next node to expand -- so the next record
//     is requested at that moment (exact, never a wrong guess) and its DRAM round trip overlaps the
//     insertions.  Consuming in ascending order also lets lowerBound fall as fast as it can: the loop
//     stops at the first candidate that no longer beats it (the hop-start admission test of the
//     single-list walk admits a superset whose tail falls off the list; the final list is identical).
//   * one insertion = two shuffles (carry from the lane below) + per-slot compare/select; equal keys
//     keep arrival order (new after old, lower lane first), the tie rule of the single-list model.
//   * shared memory per query = the table and nothing else: 28 queries per SM at M=8 (was 25).
//   * K1 fused: the table never exists in HBM.  The codebook is read from L2 through a transposed copy
//     ([m][j/V][c][V], V = 4 or 2 floats) so that a warp's codeword loads are fully coalesced.
//     The literal `tables=` call form (the reference's dtables argument) is served by the same kernel:
//     the table is then staged by one TMA bulk copy (cp.async.bulk + mbarrier) per query.
//
// Results, hop and neighbour counters are those of hnsw_walk_fast and of oracle.single_list_walk on
// every input (same list after every hop, same next node); differences from the reference itself are
// confined to exact fp32 ties, as before.
#include <math_constants.h>

#include <algorithm>

#include "annb_internal.h"
#include "tma_utils.cuh"
#include "walk4_common.cuh"

namespace {

// =====================================================================================================
// CELLS: the multi-cell (IVF) walk of annb_cellset_search.  The work item is a query: its table is built once and then
// walked over each of its probed cells in probe order (p.cells, p.cell_order; the cells share one PQ codebook), the
// results of cell c going to row q * n_cells + c of the by-cell scratch.  `g_in` is unused then.  CELLS = false is the
// single-graph walk.
template <int M, int EPL, bool CELLS>
__global__ void __launch_bounds__(w4_max_threads(M, EPL), w4_min_ctas(M, EPL)) hnsw_walk4(const GraphDev g_in, const SearchParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  // warp index through a warp reduction: the compiler then knows it is warp-uniform, keeps the table base in
  // a uniform register and folds it into the LDS address ([R + UR + imm]) -- one IADD less per lookup
  const int warp = (int)__reduce_min_sync(FULL_MASK, threadIdx.x >> 5);
  const int nwarps = blockDim.x >> 5;
  constexpr int TS = M * 256;
  constexpr int CAP = 32 * EPL;
  float *T = reinterpret_cast<float *>(smem_raw) + (size_t)warp * TS;
  uint64_t *tbar = reinterpret_cast<uint64_t *>(smem_raw + (size_t)nwarps * TS * 4) + warp;
  const bool fused = p.queries != nullptr;
  uint32_t tphase = 0;
  if (!fused) {
    if (lane == 0) mbar_init(tbar, 1);
    __syncwarp();
  }
  // per cell (CELLS): the cell's ef and k; and with them everything below that depends on the graph
  int ef = p.ef;
  int k = p.k;
  const bool lane0 = lane == 0;
  const bool stats = p.out_stats != nullptr;
  // list positions ef-1 (lowerBound once full) and ef (the slot an insertion into a full list spills to)
  int wl = (ef - 1) / EPL, ws = (ef - 1) % EPL;
  // per-lane record addressing
  bool has_slot0 = lane < g_in.maxM0;
  const uint8_t *link_base0 = g_in.rec0 + 4 * lane;
  {  // keep the per-lane base as ONE 64-bit register pair (no re-derivation from the constant bank per load)
    uint64_t t = reinterpret_cast<uint64_t>(link_base0);
    asm volatile("" : "+l"(t));
    link_base0 = reinterpret_cast<const uint8_t *>(t);
  }
  unsigned code_delta0 = (unsigned)(g_in.code_off0 + lane * (M - 4));  // from a lane's link to the same lane's code row
  uint32_t rec0_bytes = (uint32_t)g_in.rec0_bytes;
  bool has_slotu = lane < g_in.maxM;

  for (;;) {
    // next query: ONE lane bumps the work counter and the value is spread with a warp REDUCTION, not a shuffle:
    // REDUX delivers it in a uniform register, so ptxas can prove that the loop exit below is warp-uniform.
    // With `__shfl_sync(qi, 0)` it cannot, and then guards every warp-level operation of the whole loop body with
    // a BRA.DIV convergence check (31 sites, ~25 extra warp instructions per hop).
    unsigned qi = 0;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.eq.u32 p, %2, 0;\n"
        "@p atom.global.add.u32 %0, [%1], 1;\n"
        "}\n"
        : "+r"(qi)
        : "l"(p.work_counter), "r"(lane)
        : "memory");
    const int64_t q = __reduce_max_sync(FULL_MASK, qi);
    if (q >= p.B) break;
    __syncwarp();  // every lane is done with the previous query's table
    if (fused) {
      const float *qg = p.queries + q * (int64_t)(M * p.ds);
      if (p.cb_vec == 4) build_table<M, 4>(T, qg, p.cbt, p.ds, p.is_ip, p.bias, lane);
      else build_table<M, 2>(T, qg, p.cbt, p.ds, p.is_ip, p.bias, lane);
    } else {
      if (lane0) {
        mbar_expect_tx(tbar, (uint32_t)TS * 4u);
        bulk_g2s(T, p.tables + q * TS, (uint32_t)TS * 4u, tbar);
      }
      mbar_wait(tbar, tphase);
      tphase ^= 1u;
    }
    if (p.dump_tables) {  // debug export of the in-shared-memory table (parity test of the fused build)
      float *o = p.dump_tables + q * TS;
      for (int i = lane; i < TS; i += 32) o[i] = T[i];
    }

    for (int ci = 0; ci < (CELLS ? p.n_probe : 1); ci++) {
    int64_t oq = q;  // output row
    if constexpr (CELLS) {
      const int c = __ldg(p.cell_order + q * p.n_probe + ci);
      k = __ldg(p.cell_k + c);
      oq = q * p.n_cells + c;
      if (k == 0) {  // no live rows: the cell is skipped (container.py:104-105)
        if (lane0) p.out_found[oq] = 0;
        continue;
      }
      const GraphDev &gc = p.cells[c];
      ef = max(p.ef, k);  // hnswalg.h:1279
      wl = (ef - 1) / EPL;
      ws = (ef - 1) % EPL;
      has_slot0 = lane < gc.maxM0;
      uint64_t t = reinterpret_cast<uint64_t>(gc.rec0 + 4 * lane);
      asm volatile("" : "+l"(t));
      link_base0 = reinterpret_cast<const uint8_t *>(t);
      code_delta0 = (unsigned)(gc.code_off0 + lane * (M - 4));
      rec0_bytes = (uint32_t)gc.rec0_bytes;
      has_slotu = lane < gc.maxM;
    }
    const GraphDev &g = CELLS ? p.cells[__ldg(p.cell_order + q * p.n_probe + ci)] : g_in;
    // outputs start at entry (CELLS ? oq * p.cell_limit : q * k), written out at each use until the walk is done: a
    // copy hoisted above it reschedules the single-graph walk

    // ---- greedy descent maxlevel..1 (hnswalg.h:1245-1274), walk4_common.cuh ----
    int hops = 0, nbrs = 0, evals = 1;
    uint32_t cur_uk, rec;
    descend4<M>(g, T, lane, has_slotu, hops, nbrs, evals, cur_uk, rec);
    evals += 1;  // searchBaseLayerST re-scores the entry (:255)

    // ---- level 0: searchBaseLayerST as a single sorted list in registers ----
    uint32_t K[EPL], V[EPL];
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      K[e] = KEY_MAX;
      V[e] = 0xffffffffu;
    }
    if (lane0) {
      K[0] = cur_uk;
      V[0] = rec | EXP_BIT;  // the entry node is hop 0
    }
    int size = 1;
    uint32_t worst = (ef == 1) ? cur_uk : KEY_MAX;  // lowerBound (:306); "infinite" while the list is not full

    Rec<M> recA, recB;
    auto load_rec = [&](Rec<M> &r, uint32_t node) {
      const uint8_t *lp = link_base0 + (size_t)node * rec0_bytes;
      r.link = EMPTY_LINK;
#pragma unroll
      for (int i = 0; i < M / 4; i++) r.cw[i] = 0u;
      if (has_slot0) {
        r.link = __ldg(reinterpret_cast<const uint32_t *>(lp));
        load_codes<M>(r.cw, lp + code_delta0);
      }
    };
    load_rec(recA, rec);

    // One hop: `cur` holds the record of the node being expanded, `nxt` receives the record of the next one.
    // The two record register sets alternate roles (no copy, so nothing waits on a load before it is needed).
    auto hop = [&](Rec<M> &cur, Rec<M> &nxt) -> bool {
      hops++;
      // ---- nearest not-yet-expanded list entry == candidate_set.top() (:268): the next node unless this hop finds
      // something closer.  Nothing here may delay the scoring below: an L2 prefetch of this entry's record (or of
      // the one after it) would stall the in-order issue until the reduction chain that finds it has resolved,
      // and cost more than the record's lead gains (DESIGN §7) ----
      uint32_t lm = KEY_MAX;
#pragma unroll
      for (int e = 0; e < EPL; e++) lm = min(lm, K[e] | (uint32_t)((int32_t)V[e] >> 31));
      const uint32_t e2key = __reduce_min_sync(FULL_MASK, lm);
      int e2src = 0;
      uint32_t e2id = 0;
      if (e2key != KEY_MAX) {
        e2src = __ffs(__ballot_sync(FULL_MASK, lm == e2key)) - 1;
        uint32_t myid = 0;
#pragma unroll
        for (int e = EPL - 1; e >= 0; e--)
          if ((K[e] | (uint32_t)((int32_t)V[e] >> 31)) == e2key) myid = V[e] & IDM;  // lowest matching slot wins
        e2id = __shfl_sync(FULL_MASK, myid, e2src);
      }
      // expand that entry: flag it (the lowest matching slot of lane e2src)
      auto take_e2 = [&]() {
        if (lane == e2src) {
          bool done = false;
#pragma unroll
          for (int e = 0; e < EPL; e++) {
            const bool hit = !done && (K[e] | (uint32_t)((int32_t)V[e] >> 31)) == e2key;
            if (hit) V[e] |= EXP_BIT;
            done |= hit;
          }
        }
      };

      // ---- score the neighbour list: one lane = one neighbour, m sequential ----
      const bool valid = cur.link != EMPTY_LINK;
      const uint32_t uk = f2u(pq_score<M>(T, cur.cw));
      uint32_t mykey = (valid && uk < worst) ? uk : KEY_MAX;  // admission (:306) against the hop-start lowerBound
      if (stats) {
        const int nv = __popc(__ballot_sync(FULL_MASK, valid));
        nbrs += nv;
        evals += nv;
      }

      // re-encounter of a listed node?  (an id can only be listed under this very key)
      auto listed = [&](uint32_t id) -> bool {
        bool dup = false;
#pragma unroll
        for (int e = 0; e < EPL; e++) dup |= (V[e] & IDM) == id;
        return __any_sync(FULL_MASK, dup);
      };

      // ---- phase A: the smallest NEW candidate (if any) against the nearest unexpanded entry: the next node is
      // known exactly, before anything is merged ----
      bool have_new = false;
      uint32_t mn, id = 0;
      for (;;) {
        mn = __reduce_min_sync(FULL_MASK, mykey);
        if (mn == KEY_MAX) break;  // none (left) that beats lowerBound
        const int src = __ffs(__ballot_sync(FULL_MASK, mykey == mn)) - 1;  // lower lane first among equals
        id = __shfl_sync(FULL_MASK, cur.link, src);
        if (lane == src) mykey = KEY_MAX;
        if (!listed(id)) {
          have_new = true;
          break;
        }
      }
      if (have_new && mn < e2key) {
        load_rec(nxt, id);  // replaces the guess; its DRAM round trip overlaps the insertions below
        list_insert<EPL>(K, V, mn, id | EXP_BIT, lane0);
        size++;
      } else {
        if (e2key == KEY_MAX) return false;  // nothing unexpanded and nothing new: candidate_set exhausted (:266)
        load_rec(nxt, e2id);
        take_e2();
        if (have_new) {
          list_insert<EPL>(K, V, mn, id, lane0);
          size++;
        }
      }
      // ---- phase B: the other admitted candidates in lane order (equal keys keep arrival order).  lowerBound
      // is NOT refreshed per insertion: a candidate that the falling bound would have rejected lands at a
      // position >= ef and drops out below, exactly like the hop-start admission rule of the single-list walk ----
      if (have_new) {
        // (A/B, round 2: checking the re-encounters of a hop four at a time ahead of the insertions, with the next
        // candidate's key/id fetched before the current insertion, was 13 % SLOWER -- 30.4 vs 34.8 M QPS on one box:
        // the padded groups cost more issue slots than the overlapped latencies give back at ~3.4 candidates per hop)
        unsigned live = __ballot_sync(FULL_MASK, mykey != KEY_MAX);
        while (live) {
          const int src = __ffs(live) - 1;
          live &= live - 1;
          const uint32_t ck = __shfl_sync(FULL_MASK, mykey, src);
          const uint32_t cid = __shfl_sync(FULL_MASK, cur.link, src);
          if (listed(cid)) continue;
          list_insert<EPL>(K, V, ck, cid, lane0);
          size++;
        }
        if (size >= ef) {
          size = ef;
          worst = list_key_at<EPL>(K, wl, ws);  // lowerBound = top_candidates.top() (:320-321)
          if (ef < CAP) {                        // what spilled past position ef-1 is gone
#pragma unroll
            for (int e = 0; e < EPL; e++)
              if (lane * EPL + e >= ef) {
                K[e] = KEY_MAX;
                V[e] = 0xffffffffu;
              }
          }
        }
      }
      return true;
    };
    for (;;) {
      if (!hop(recA, recB)) break;
      if (!hop(recB, recA)) break;
    }

    // ---- results: the first k list entries, ascending (dist, label) (hnsw_bindings.cpp:346-351) ----
    const int64_t row = CELLS ? oq * p.cell_limit : q * k;
    const int found = min(size, k);
    bool tie = false;
    const uint32_t k_next_lane = __shfl_down_sync(FULL_MASK, K[0], 1);
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const int pos = lane * EPL + e;
      if (pos < k) {
        const bool have = pos < size;
        p.out_dists[row + pos] = have ? u2f(K[e]) : CUDART_INF_F;
        p.out_labels[row + pos] = have ? (p.out_internal ? (uint64_t)(V[e] & IDM) : __ldg(g.labels + (V[e] & IDM))) : (uint64_t)UINT64_MAX;
      }
      const uint32_t nk = (e + 1 < EPL) ? K[e + 1 < EPL ? e + 1 : e] : k_next_lane;
      tie |= (pos + 1 < found) && (nk == K[e]) && (e + 1 < EPL || lane < 31);
    }
    if (__any_sync(FULL_MASK, tie)) {
      __syncwarp();
      if (lane0) sort_ties(p, row, found);
    }
    if (lane0) {
      p.out_found[oq] = found;
      if (stats) {
        p.out_stats[oq * 3 + 0] = hops;
        p.out_stats[oq * 3 + 1] = nbrs;
        p.out_stats[oq * 3 + 2] = evals;
      }
    }
    }
  }
}

template <int M, bool CELLS>
int launch_walk4_m(annb_index *h, const SearchParams &p, int ef) {
  return with_epl(ef, [&](auto epl) {  // the callers hold ef to ANNB_MAX_EF
    constexpr int EPL = decltype(epl)::value;
    return launch_w4<M, EPL>(h, hnsw_walk4<M, EPL, CELLS>, p);
  });
}

}  // namespace

// Can the plain (no filter, no deletions) search of this index run on hnsw_walk4 at all?
bool walk4_applicable(const annb_index *h) {
  if (h->opt_walk_kernel == 1) return false;  // A/B switch: force the round-1 kernels
  const GraphDev &d = h->gd;
  return h->Ks == 256 && h->code_bytes == 1 && (h->M == 8 || h->M == 16 || h->M == 32) && d.maxM0 <= 32 && d.maxM <= 32 &&
         d.n < 0x7fffffffll;
}

// ... and may it build the tables itself from the queries (fused K1)?  Needs a vectorisable subvector
// length and a staging layout that is consumed before it is overwritten (see build_table).
bool walk4_can_fuse(const annb_index *h) {
  if (h->opt_walk_kernel == 2) return false;  // A/B switch: hnsw_walk4 on materialised tables
  if (!walk4_applicable(h) || !h->d_codebook_t || h->cb_vec == 0) return false;
  const int M = h->M, ds = h->ds, D = M * ds;
  const int R = (D + 255) / 256;
  if (R > M) return false;
  for (int t = 0; t + 1 < R; t++)
    if ((t + 1) * 256 > (M - R + t + 1) * ds) return false;
  return true;
}

int launch_walk4(annb_index *h, const SearchParams &p) {
  if (p.B == 0) return ANNB_OK;
  if (!p.queries && (reinterpret_cast<uintptr_t>(p.tables) & 15)) return 1;  // TMA needs 16-byte alignment
  if (p.ef > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "ef=%d exceeds ANNB_MAX_EF=%d", p.ef, ANNB_MAX_EF);
  switch (h->M) {
    case 8: return launch_walk4_m<8, false>(h, p, p.ef);
    case 16: return launch_walk4_m<16, false>(h, p, p.ef);
    case 32: return launch_walk4_m<32, false>(h, p, p.ef);
  }
  return 1;
}

// The multi-cell walk: p.ef = the caller's ef (cell c walks with max(ef, k_c)), p.cell_limit = the largest k_c; h = the
// handle whose stream and scratch the launch uses.  Only the fused table build (p.queries) and M = 8 are instantiated: the cell set routes every other
// geometry to its generic per-cell route.
int launch_walk4_cells(annb_index *h, const SearchParams &p) {
  if (p.B == 0) return ANNB_OK;
  if (!p.queries || h->M != 8) return 1;
  const int ef_max = std::max(p.ef, p.cell_limit);  // the largest max(ef, k_c) of any cell sizes the list
  if (ef_max > ANNB_MAX_EF) ANNB_FAIL(ANNB_ELIMIT, "max(ef, limit)=%d exceeds ANNB_MAX_EF=%d", ef_max, ANNB_MAX_EF);
  return launch_walk4_m<8, true>(h, p, ef_max);
}
