// walk_flagged4.cu -- the filtered / deletion-aware search in hnsw_walk4's machine mapping: K1 inside the kernel
// (table built in shared memory, or TMA-staged for the literal `tables=` form), everything else in registers.
//
// Reference semantics:
//   searchKnnWithFilter  include/hnswlib/hnswalg.h:1297-1361 -> searchBaseLayerSTWithFilter :332-440
//   searchKnn with deleted nodes :1237-1295 -> searchBaseLayerST<true> :243-329
//   binding: knn_query_with_filter  bindings/hnsw_bindings.cpp:393-516
//
// hnsw_walk_flagged (hnsw_search.cu) keeps every evaluated node the reference would push to candidate_set in ONE
// sorted list with a PASS flag; at a 50 % filter that list is 4x the plain search's and lives in a shared-memory
// mirror (CAP = 256: 1.49 ms per 10 000 queries at configs[3]; a single REGISTER list of that length was measured
// slower still, 1.87 ms, because one insertion touches all 8 slots of every lane).  Here the same set is kept as TWO
// register lists:
//   P  the admitted entries (pass the filter / not deleted) = top_candidates, at most ef of them -- exactly the
//      list of hnsw_walk4, same length, same insertion;
//   N  the traversed-but-not-admitted entries = the members of candidate_set that are not in top_candidates.
// An insertion goes to ONE of them (the pass bit of the candidate is warp-uniform), so it costs what it costs in the
// plain search.  lowerBound (top_candidates.top()) is P's ef-th key once P is full, else P's largest key, else
// FLT_MAX (:256-260 / :353-360).  N entries beyond lowerBound are never expanded (the loop breaks first, :270 / :371);
// they are not pruned either -- N simply keeps its 32*EN smallest entries, so what falls off its end when it is full
// are those dead entries first.  While P is not full nothing may be lost -- which is what makes the walk exact
// without a visited set (a re-encountered node is still listed, or was lost with d > a lowerBound that has only
// fallen since and fails the admission test).  The next node is the nearest unexpanded entry of either list or a
// closer new candidate; the break rules are the reference's: with a filter `d > lowerBound` alone (:371, no size
// guard), with deletions `d > lowerBound && (size == ef || !has_deletions)` (:270).
//
// N's capacity (32*EN) is chosen by the host from the selectivity.  Lane 31 tracks the smallest key that ever fell off
// N's end; the query is flagged (found = -1) only if such an entry could still have mattered (P not full, or its key
// <= lowerBound) and the host re-runs exactly those queries on the bitmap walk.
//
// Instruction diet (ncu, first version: 435 warp instructions per hop, ALU pipe 83 % busy): the nearest unexpanded
// entry is tracked as a per-lane (key, value) minimum and flagged by id (was: key scan + slot search + flag search,
// 13 instructions per slot); the re-encounter check compares KEYS first and ids only when a key matches; N is not
// pruned per hop.
//
// Differences from the reference are confined to exact fp32 ties (arrival order instead of heap order), as for
// every single-list walk here; tests/test_gpu_walk4f.py checks ids, distance bits, hop and neighbour counts against
// the oracle on every tie-free walk, tests/test_walk_model.py the scalar model of this walk (oracle.two_list_walk)
// against the restatement of the reference on the CPU.
#include <math_constants.h>

#include <algorithm>

#include "annb_internal.h"
#include "tma_utils.cuh"
#include "walk4_common.cuh"

namespace {

constexpr uint32_t KEY_FLT_MAX = 0xff7fffffu;  // f2u(FLT_MAX): lowerBound while nothing is admitted (:260)

// PQF (per-query filter): query q is admitted by the bitmap p.query_filter[q] (nullptr = "not deleted") instead of the
// launch's one p.filter; the choice is made at the start of each query.  PQF = false is the single-filter walk.
//
// CELLS: the filtered multi-cell (IVF) walk of annb_cellset_search_prepared, hnsw_walk4<M, EPL, true>'s work mapping.
// The work item is a query: its table is built once and then walked over each of its probed cells in probe order
// (p.cells, p.cell_order), cell c admitting by its own prepared bitmap p.cell_filter[c] (filter semantics in every cell:
// no size guard) with k_c = p.cell_k[c] (0 = skip the cell) and ef_c = max(ef, k_c).  Results, found and counters go to
// row q * n_cells + c of the by-cell scratch; a (query, cell) walk that outgrows N writes found = -1 for that pair only
// and the query goes on with its next cell.  `g_in` and `has_del` are unused then.
//
// PQF and CELLS: the per-query filtered multi-cell walk of annb_cellset_search_multi.  Query q belongs to slot
// s = p.query_slot[q] (queries with the same filter in every cell share one); cell c is walked with the pair's
// k = p.cell_k[s * n_cells + c] (0 = skip) and admission word p.cell_filter[s * n_cells + c], a bitmap pointer whose
// low bits say how to read it: bit 0 = "not deleted" (flip, the query has no filter in this cell: the bitmap is the
// cell's deletions), bit 1 = the size guard of :270 (the cell has deletions).  Without either bit it is a prepared
// filter with filter semantics, as in the CELLS form.
//
// Launch geometry: hnsw_walk4's EPL <= 4 shape (walk4_common.cuh).
template <int M, int EP, int EN, bool PQF, bool CELLS>
__global__ void __launch_bounds__(w4_max_threads(M, 4), w4_min_ctas(M, 4))
    hnsw_walk4f(const GraphDev g_in, const SearchParams p, const int has_del) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = (int)__reduce_min_sync(FULL_MASK, threadIdx.x >> 5);  // uniform register (see hnsw_walk4)
  const int nwarps = blockDim.x >> 5;
  constexpr int TS = M * 256;
  constexpr int CAPP = 32 * EP;
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
  int wl = (ef - 1) / EP, ws = (ef - 1) % EP;  // P's position ef-1: lowerBound once P is full
  // admission bit by internal id: the filter bitmap (:353-354, :423-426; delete marks are ignored under a filter),
  // else "not deleted" (:254, :314)
  bool use_filter = p.filter != nullptr;
  const uint32_t *__restrict__ bits = use_filter ? p.filter : g_in.deleted;
  uint32_t flip = use_filter ? 0u : 1u;
  auto passes = [&](uint32_t id) -> uint32_t { return ((__ldg(bits + (id >> 5)) >> (id & 31)) & 1u) ^ flip; };
  bool size_guard = !use_filter && has_del;  // :270 breaks only when top_candidates is full; :371 has no such guard
  if constexpr (CELLS) {  // every cell admits by its own bitmap (set per cell below)
    use_filter = true;
    flip = 0u;
    size_guard = false;
  }

  bool has_slot0 = lane < g_in.maxM0;
  const uint8_t *link_base0 = g_in.rec0 + 4 * lane;
  {
    uint64_t t = reinterpret_cast<uint64_t>(link_base0);
    asm volatile("" : "+l"(t));
    link_base0 = reinterpret_cast<const uint8_t *>(t);
  }
  unsigned code_delta0 = (unsigned)(g_in.code_off0 + lane * (M - 4));
  uint32_t rec0_bytes = (uint32_t)g_in.rec0_bytes;
  bool has_slotu = lane < g_in.maxM;

  for (;;) {
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
    __syncwarp();
    if constexpr (PQF && !CELLS) {
      const uint32_t *f = p.query_filter[q];
      use_filter = f != nullptr;
      bits = use_filter ? f : g_in.deleted;
      flip = use_filter ? 0u : 1u;
      size_guard = !use_filter && has_del;
    }
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
    if (p.dump_tables) {
      float *o = p.dump_tables + q * TS;
      for (int i = lane; i < TS; i += 32) o[i] = T[i];
    }

    int slot_row = 0;  // PQF && CELLS: first entry of the query's slot in the (slot, cell) tables
    if constexpr (PQF && CELLS) slot_row = __ldg(p.query_slot + q) * p.n_cells;
    for (int ci = 0; ci < (CELLS ? p.n_probe : 1); ci++) {
    int64_t oq = q;  // output row
    if constexpr (CELLS) {
      const int c = __ldg(p.cell_order + q * p.n_probe + ci);
      if constexpr (PQF) k = __ldg(p.cell_k + slot_row + c);
      else k = __ldg(p.cell_k + c);
      oq = q * p.n_cells + c;
      if (k == 0) {  // nothing admitted: the cell is skipped
        if (lane0) p.out_found[oq] = 0;
        continue;
      }
      const GraphDev &gc = p.cells[c];
      ef = max(p.ef, k);  // hnswalg.h:1279
      wl = (ef - 1) / EP;
      ws = (ef - 1) % EP;
      if constexpr (PQF) {
        const uintptr_t w = reinterpret_cast<uintptr_t>(p.cell_filter[slot_row + c]);
        bits = reinterpret_cast<const uint32_t *>(w & ~(uintptr_t)3);
        flip = (uint32_t)(w & 1u);
        size_guard = (w & 2u) != 0;
      } else {
        bits = p.cell_filter[c];
      }
      has_slot0 = lane < gc.maxM0;
      uint64_t t = reinterpret_cast<uint64_t>(gc.rec0 + 4 * lane);
      asm volatile("" : "+l"(t));
      link_base0 = reinterpret_cast<const uint8_t *>(t);
      code_delta0 = (unsigned)(gc.code_off0 + lane * (M - 4));
      rec0_bytes = (uint32_t)gc.rec0_bytes;
      has_slotu = lane < gc.maxM;
    }
    const GraphDev &g = CELLS ? p.cells[__ldg(p.cell_order + q * p.n_probe + ci)] : g_in;
    // outputs start at entry (CELLS ? oq * p.cell_limit : q * k), computed after the walk as in hnsw_walk4

    int hops = 0, nbrs = 0, evals = 1;
    uint32_t cur_uk, rec;
    descend4<M>(g, T, lane, has_slotu, hops, nbrs, evals, cur_uk, rec);
    evals += 1;

    // ---- level 0: top_candidates = P, candidate_set \ top_candidates = N ----
    uint32_t KP[EP], VP[EP], KN[EN], VN[EN];
#pragma unroll
    for (int e = 0; e < EP; e++) {
      KP[e] = KEY_MAX;
      VP[e] = 0xffffffffu;
    }
#pragma unroll
    for (int e = 0; e < EN; e++) {
      KN[e] = KEY_MAX;
      VN[e] = 0xffffffffu;
    }
    const bool ep_pass = passes(rec) != 0u;  // :254 / :353
    if (lane0) {
      if (ep_pass) {
        KP[0] = cur_uk;
        VP[0] = rec | EXP_BIT;
      } else {
        KN[0] = cur_uk;
        VN[0] = rec | EXP_BIT;
      }
    }
    int sizeP = ep_pass ? 1 : 0;
    uint32_t pmax = ep_pass ? cur_uk : 0u;                 // largest admitted key while P is not full
    uint32_t lb = ep_pass ? cur_uk : KEY_FLT_MAX;          // lowerBound (:256 / :260)
    uint32_t worst = (sizeP >= ef) ? lb : KEY_MAX;         // admission bound (:306 / :413): none while P is not full
    uint32_t lost = KEY_MAX;                               // lane 31: smallest key that fell off N's end
    bool aborted = false;

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

    auto hop = [&](Rec<M> &cur, Rec<M> &nxt) -> bool {
      hops++;
      // admission bits of this node's neighbours: issued first, consumed after the scores
      const bool valid = cur.link != EMPTY_LINK;
      uint32_t pf = 0u;
      if (valid) pf = passes(cur.link);

      // ---- nearest not-yet-expanded entry of either list == candidate_set.top() (:268 / :369): every lane keeps
      // the (key, value) of its own nearest one (lowest slot among equals, P before N), one REDUX picks the lane ----
      uint32_t lm = KEY_MAX, lv = 0u;
      unexpanded_min<EP>(KP, VP, lm, lv);
      unexpanded_min<EN>(KN, VN, lm, lv);
      const uint32_t e2key = __reduce_min_sync(FULL_MASK, lm);
      uint32_t e2id = 0;
      if (e2key != KEY_MAX) {
        const int e2src = __ffs(__ballot_sync(FULL_MASK, lm == e2key)) - 1;
        e2id = __shfl_sync(FULL_MASK, lv, e2src);  // (an unexpanded entry's value is its node id: no flag bit set)
      }
      // expand that entry: ids are unique in the lists and an unexpanded entry's value IS its id
      auto take_e2 = [&]() {
#pragma unroll
        for (int e = 0; e < EP; e++)
          if (VP[e] == e2id) VP[e] |= EXP_BIT;
#pragma unroll
        for (int e = 0; e < EN; e++)
          if (VN[e] == e2id) VN[e] |= EXP_BIT;
      };

      // ---- score the neighbour list: one lane = one neighbour, m sequential ----
      const uint32_t uk = f2u(pq_score<M>(T, cur.cw));
      uint32_t mykey = (valid && uk < worst) ? uk : KEY_MAX;
      if (stats) {
        const int nv = __popc(__ballot_sync(FULL_MASK, valid));
        nbrs += nv;
        evals += nv;
      }

      // re-encounter of a listed node?  An id can only be listed under this very key, so the id compare runs only
      // when some entry has an equal key (a re-encounter, or an exact fp32 tie between two nodes)
      auto listed = [&](uint32_t key, uint32_t id) -> bool {
        bool eq = false;
#pragma unroll
        for (int e = 0; e < EP; e++) eq |= KP[e] == key;
#pragma unroll
        for (int e = 0; e < EN; e++) eq |= KN[e] == key;
        if (!__any_sync(FULL_MASK, eq)) return false;
        bool dup = false;
#pragma unroll
        for (int e = 0; e < EP; e++) dup |= (VP[e] & IDM) == id;
#pragma unroll
        for (int e = 0; e < EN; e++) dup |= (VN[e] & IDM) == id;
        return __any_sync(FULL_MASK, dup);
      };
      // one insertion: into P (admitted) or N (traversed only); `pass` is warp-uniform
      auto insert = [&](uint32_t key, uint32_t val, bool pass) {
        if (pass) {
          list_insert<EP>(KP, VP, key, val, lane0);
          sizeP++;
          pmax = max(pmax, key);
        } else {
          const uint32_t last = KN[EN - 1];  // (lane 31's is N's last position)
          if (last != KEY_MAX) lost = min(lost, max(last, key));
          list_insert<EN>(KN, VN, key, val, lane0);
        }
      };

      // ---- phase A: the smallest NEW candidate against the nearest unexpanded entry: the next node, exactly ----
      bool have_new = false;
      uint32_t mn, id = 0;
      int src = 0;
      for (;;) {
        mn = __reduce_min_sync(FULL_MASK, mykey);
        if (mn == KEY_MAX) break;
        src = __ffs(__ballot_sync(FULL_MASK, mykey == mn)) - 1;
        id = __shfl_sync(FULL_MASK, cur.link, src);
        if (lane == src) mykey = KEY_MAX;
        if (!listed(mn, id)) {
          have_new = true;
          break;
        }
      }
      const bool new_is_next = have_new && mn < e2key;
      if (!new_is_next && e2key == KEY_MAX) return false;  // candidate_set exhausted (:266 / :367)
      load_rec(nxt, new_is_next ? id : e2id);  // requested BEFORE the admission bits are waited for: the two round trips overlap
      if (!new_is_next) take_e2();
      const uint32_t nextkey = new_is_next ? mn : e2key;
      const unsigned passmask = __ballot_sync(FULL_MASK, pf != 0u);
      if (have_new) insert(mn, new_is_next ? (id | EXP_BIT) : id, (passmask >> src) & 1u);
      // ---- phase B: the other admitted candidates in lane order ----
      if (have_new) {
        unsigned live = __ballot_sync(FULL_MASK, mykey != KEY_MAX);
        while (live) {
          const int s2 = __ffs(live) - 1;
          live &= live - 1;
          const uint32_t ck = __shfl_sync(FULL_MASK, mykey, s2);
          const uint32_t cid = __shfl_sync(FULL_MASK, cur.link, s2);
          if (listed(ck, cid)) continue;
          insert(ck, cid, (passmask >> s2) & 1u);
        }
        // ---- lowerBound = top_candidates.top() (:320-321 / :429-430) ----
        if (sizeP >= ef) {
          sizeP = ef;
          lb = list_key_at<EP>(KP, wl, ws);
          worst = lb;
          if (ef < CAPP) {
#pragma unroll
            for (int e = 0; e < EP; e++)
              if (lane * EP + e >= ef) {
                KP[e] = KEY_MAX;
                VP[e] = 0xffffffffu;
              }
          }
          // (N is not pruned: entries beyond lowerBound are never expanded -- the break rule below ends the walk
          // before -- and they are the first to fall off N's end when it is full)
        } else if (sizeP > 0) {
          lb = pmax;
        }
        const uint32_t lostv = __shfl_sync(FULL_MASK, lost, 31);
        if (lostv != KEY_MAX && !(sizeP >= ef && lostv > lb)) {
          aborted = true;  // an entry that could still be expanded fell off N: the host re-runs this query
          return false;
        }
      }
      // ---- break rule on the node about to be expanded (:270 / :371) ----
      if (nextkey > lb && (!size_guard || sizeP >= ef)) return false;
      return true;
    };
    for (;;) {
      if (!hop(recA, recB)) break;
      if (!hop(recB, recA)) break;
    }

    if (aborted) {
      if (lane0) p.out_found[oq] = -1;
      continue;
    }
    // ---- results: the first k admitted entries, ascending (dist, label) (hnsw_bindings.cpp:346-351) ----
    const int64_t row = CELLS ? oq * p.cell_limit : q * k;
    const int found = min(min(sizeP, ef), k);
    bool tie = false;
    const uint32_t k_next_lane = __shfl_down_sync(FULL_MASK, KP[0], 1);
#pragma unroll
    for (int e = 0; e < EP; e++) {
      const int pos = lane * EP + e;
      if (pos < k) {
        const bool have = pos < found;
        p.out_dists[row + pos] = have ? u2f(KP[e]) : CUDART_INF_F;
        p.out_labels[row + pos] = have ? (p.out_internal ? (uint64_t)(VP[e] & IDM) : __ldg(g.labels + (VP[e] & IDM))) : (uint64_t)UINT64_MAX;
      }
      const uint32_t nk = (e + 1 < EP) ? KP[e + 1 < EP ? e + 1 : e] : k_next_lane;
      tie |= (pos + 1 < found) && (nk == KP[e]) && (e + 1 < EP || lane < 31);
    }
    for (int r = CAPP + lane; r < k; r += 32) {  // k > 32*EP cannot happen (ef >= k, CAPP >= ef); kept for safety
      p.out_dists[row + r] = CUDART_INF_F;
      p.out_labels[row + r] = (uint64_t)UINT64_MAX;
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

template <int M, int EP, int EN, bool CELLS>
int launch_walk4f_t(annb_index *h, const SearchParams &p) {
  void (*kern)(const GraphDev, const SearchParams, const int);
  if constexpr (CELLS) kern = p.query_slot ? hnsw_walk4f<M, EP, EN, true, true> : hnsw_walk4f<M, EP, EN, false, true>;
  else kern = p.query_filter ? hnsw_walk4f<M, EP, EN, true, false> : hnsw_walk4f<M, EP, EN, false, false>;
  return launch_w4<M, 4>(h, kern, p, h->g.num_deleted > 0 ? 1 : 0);
}

// f(EP, EN) as std::integral_constant for the instantiated list geometries (walk4f_geometry gives no others); 1 = none
template <typename F>
int with_ep_en(int ep, int en, F f) {
  using std::integral_constant;
  if (ep == 2) {
    switch (en) {
      case 2: return f(integral_constant<int, 2>(), integral_constant<int, 2>());
      case 3: return f(integral_constant<int, 2>(), integral_constant<int, 3>());
      case 4: return f(integral_constant<int, 2>(), integral_constant<int, 4>());
      case 5: return f(integral_constant<int, 2>(), integral_constant<int, 5>());
      case 6: return f(integral_constant<int, 2>(), integral_constant<int, 6>());
      case 8: return f(integral_constant<int, 2>(), integral_constant<int, 8>());
    }
  } else if (ep == 4) {
    switch (en) {
      case 4: return f(integral_constant<int, 4>(), integral_constant<int, 4>());
      case 6: return f(integral_constant<int, 4>(), integral_constant<int, 6>());
      case 8: return f(integral_constant<int, 4>(), integral_constant<int, 8>());
    }
  }
  return 1;
}

template <int M, bool CELLS>
int launch_walk4f_m(annb_index *h, const SearchParams &p, int ep, int en) {
  return with_ep_en(ep, en, [&](auto ep_c, auto en_c) {
    return launch_walk4f_t<M, decltype(ep_c)::value, decltype(en_c)::value, CELLS>(h, p);
  });
}

}  // namespace

// N's capacity for a filter (or deletion rate) that admits a fraction s of the nodes.  While P holds fewer than ef
// entries N must keep every rejected node that was evaluated: a negative-binomial count with mean ef(1-s)/s and
// variance ef(1-s)/s^2; afterwards it must keep the rejected nodes below lowerBound -- the same count again, but it is
// the MAXIMUM of that count over the ~150 hops of a walk that has to fit.  Measured with the scalar model
// (oracle.two_list_walk, ef = 64, s = 0.5: mean 64, sigma 11.3): the per-walk maximum has mean 77-84 and reached 123
// in 3 000 walks, so mean + 4.5 sigma (128 entries) flags a query in every few thousand; mean + 6.5 sigma does not.
static int walk4f_en_for(int ef, double s) {
  s = std::min(1.0, std::max(1e-4, s));
  const double mean = ef * (1.0 - s) / s, sd = std::sqrt(ef * (1.0 - s)) / s;
  const double need = mean + 6.5 * sd + 4.0;
  for (int en : {2, 3, 4, 5, 6, 8})
    if (en * 32 >= need) return en;
  return 0;
}

// Can this filtered / deletion-aware search run on the two-list kernel?  (ep, en) = entries per lane of P and N.
bool walk4f_geometry(const annb_index *h, int ef, double selectivity, int *ep_out, int *en_out) {
  if (h->opt_flagged_kernel == 1 || h->opt_flagged_epl > 0) return false;  // A/B and test switches: hnsw_walk_flagged
  if (!walk4_applicable(h) || h->gd.n >= (1ll << 30)) return false;
  if (ef > 128) return false;  // P wider than 4 entries per lane: the shared-memory merge of hnsw_walk_flagged
  const int ep = ef <= 64 ? 2 : 4;
  int en = walk4f_en_for(ef, selectivity);
  if (h->opt_flagged_en >= 2 && h->opt_flagged_en <= 8 && h->opt_flagged_en != 7) en = (int)h->opt_flagged_en;  // tests / A-B: force N's size
  if (en == 0) return false;
  *ep_out = ep;
  *en_out = walk4f_round_en(ep, en);
  return true;
}
int walk4f_round_en(int ep, int en) { return ep == 4 ? (en <= 4 ? 4 : (en <= 6 ? 6 : 8)) : en; }
bool walk4f_applicable(const annb_index *h, int ef, double selectivity) {
  int ep, en;
  return walk4f_geometry(h, ef, selectivity, &ep, &en);
}

// filtered / deletion-aware search on the two-list kernel; returns 1 = not applicable (caller takes hnsw_walk_flagged)
int launch_walk4f(annb_index *h, const SearchParams &p) {
  if (p.B == 0) return ANNB_OK;
  int ep, en;
  if (!walk4f_geometry(h, p.ef, (double)p.selectivity, &ep, &en)) return 1;
  if (!p.queries && (!p.tables || (reinterpret_cast<uintptr_t>(p.tables) & 15))) return 1;
  switch (h->M) {
    case 8: return launch_walk4f_m<8, false>(h, p, ep, en);
    case 16: return launch_walk4f_m<16, false>(h, p, ep, en);
    case 32: return launch_walk4f_m<32, false>(h, p, ep, en);
  }
  return 1;
}

// The filtered multi-cell walk (hnsw_walk4f<8, EP, EN, false, true>): p.ef = the caller's ef, p.cell_limit = the row
// length of the scratch (>= every k_c), (ep, en) = the lists' entries per lane as walk4f_geometry gives them, chosen by
// the caller to cover every walked cell; h = the handle whose stream and scratch the launch uses.  Only the fused table
// build and M = 8 are instantiated.  With p.query_slot set, the per-query form (hnsw_walk4f<8, EP, EN, true, true>):
// p.cell_k and p.cell_filter are then (slots, n_cells) tables.
int launch_walk4f_cells(annb_index *h, const SearchParams &p, int ep, int en) {
  if (p.B == 0) return ANNB_OK;
  if (!p.queries || h->M != 8 || !p.cell_filter) return 1;
  return launch_walk4f_m<8, true>(h, p, ep, en);
}
