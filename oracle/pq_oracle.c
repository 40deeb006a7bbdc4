/*
 * pq_oracle.c -- CPU restatement of the reference's PQ-ADC / PQ-HNSW search path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under annlite_b200/ may call, link or import this file;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do,
 * and only as the checker.  The shipped path is CUDA and fails loudly without its extension.
 *
 * Parity status: PINNED.  The reference holds no golden vectors for this path (SURVEY.md 8c),
 * so the restatement is pinned against outputs of the reference itself, compiled from
 * /root/reference by oracle/build_ref.py (oracle/_ref) -- see tests/test_oracle_vs_ref.py (runs
 * where oracle/_ref exists) and the committed fixtures in tests/golden/ made by
 * oracle/make_golden.py from that same compiled reference.  Ids AND fp32 distances are
 * bit-identical, including tie behaviour, because the std::priority_queue heap moves of
 * libstdc++ (bits/stl_heap.h: __push_heap / __adjust_heap) are restated exactly below.
 *
 * Build:  gcc -O2 -std=c11 -ffp-contract=off -fPIC -shared  (no FMA: the reference is built with
 *         -std=c++14 => ISO mode => -ffp-contract=off, setup.py:108-119,151).
 *
 * Every function cites the reference file:line it follows (paths relative to /root/reference).
 *
 * The functions from orc_single_list_walk on are the exception and are marked as such: scalar models of
 * the PRODUCT's walks and of its batched GPU build's back-links, run beside the restatement by tests.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------ */
/* ADC tables                                                                                 */
/* ------------------------------------------------------------------------------------------ */

/* bindings/pq_bindings.pyx:149-210 (batch) and :85-145 (single query = B==1):
 * T[b,m,c] = sum_j (cb[m,c,j] - q[b,m*ds+j])^2, j strictly sequential, sub/mul/add each rounded. */
ORC_API void orc_adc_table_l2(const float *q, const float *cb, int64_t B, int M, int Ks, int ds,
                              float *out) {
  const int D = M * ds;
  for (int64_t b = 0; b < B; b++)
    for (int m = 0; m < M; m++)
      for (int c = 0; c < Ks; c++) {
        const float *w = cb + ((size_t)m * Ks + c) * ds;
        const float *x = q + (size_t)b * D + (size_t)m * ds;
        float acc = 0.f;
        for (int j = 0; j < ds; j++) {
          float coord = w[j] - x[j];
          acc += coord * coord;
        }
        out[((size_t)b * M + m) * Ks + c] = acc;
      }
}

/* bindings/pq_bindings.pyx:214-274 then annlite/core/codec/pq.py:316-322:
 * T[b,m,c] = fp32(1/Ks) - sum_j cb[m,c,j]*q[b,m*ds+j]  (numpy: python float is a weak scalar,
 * so `1/Ks - float32_array` is an fp32 subtraction with 1/Ks rounded to fp32 first). */
ORC_API void orc_adc_table_ip(const float *q, const float *cb, int64_t B, int M, int Ks, int ds,
                              float *out) {
  const int D = M * ds;
  const float bias = (float)(1.0 / (double)Ks);
  for (int64_t b = 0; b < B; b++)
    for (int m = 0; m < M; m++)
      for (int c = 0; c < Ks; c++) {
        const float *w = cb + ((size_t)m * Ks + c) * ds;
        const float *x = q + (size_t)b * D + (size_t)m * ds;
        float acc = 0.f;
        for (int j = 0; j < ds; j++) acc += w[j] * x[j];
        out[((size_t)b * M + m) * Ks + c] = bias - acc;
      }
}

/* ------------------------------------------------------------------------------------------ */
/* One ADC distance and the exhaustive scan                                                   */
/* ------------------------------------------------------------------------------------------ */

/* include/hnswlib/space_pq.h:16-37 (PQLookup) == bindings/pq_bindings.pyx:30-47:
 * d = sum_m T[m, code[m]], m strictly sequential, starting from 0.f. */
static inline float pq_lookup(const float *table, int M, int Ks, const uint8_t *code, int code_bytes) {
  float res = 0.f;
  for (int i = 0; i < M; i++) {
    uint32_t c;
    if (code_bytes == 1) c = code[i];
    else if (code_bytes == 2) { uint16_t t; memcpy(&t, code + 2 * i, 2); c = t; }
    else { memcpy(&c, code + 4 * i, 4); }
    res += table[(size_t)i * Ks + c];
  }
  return res;
}

/* bindings/pq_bindings.pyx:52-80 (dist_pqcodes_to_codebooks): one table, all N codes. */
ORC_API void orc_scan(const float *table, const void *codes, int64_t N, int M, int Ks, int code_bytes,
                      float *out) {
  const uint8_t *c = (const uint8_t *)codes;
  for (int64_t n = 0; n < N; n++) out[n] = pq_lookup(table, M, Ks, c + (size_t)n * M * code_bytes, code_bytes);
}

/* annlite/core/index/pq_index.py:29-56 + annlite/math.py:94-120: k smallest of the scan, ascending.
 * numpy's argpartition/argsort leave the order of equal distances unspecified; the restatement
 * fixes it as (distance, index) and the parity tests are tie-aware.  Simple O(N*k) insertion. */
ORC_API void orc_scan_topk(const float *tables, const void *codes, int64_t B, int64_t N, int M, int Ks,
                           int code_bytes, int k, int64_t *ids, float *dists) {
  const uint8_t *c = (const uint8_t *)codes;
  for (int64_t b = 0; b < B; b++) {
    const float *t = tables + (size_t)b * M * Ks;
    float *bd = dists + (size_t)b * k;
    int64_t *bi = ids + (size_t)b * k;
    int cnt = 0;
    for (int64_t n = 0; n < N; n++) {
      float d = pq_lookup(t, M, Ks, c + (size_t)n * M * code_bytes, code_bytes);
      if (cnt == k && !(d < bd[k - 1])) continue; /* later index loses ties */
      int p = cnt < k ? cnt : k - 1;
      while (p > 0 && bd[p - 1] > d) { bd[p] = bd[p - 1]; bi[p] = bi[p - 1]; p--; }
      bd[p] = d; bi[p] = n;
      if (cnt < k) cnt++;
    }
    for (int j = cnt; j < k; j++) { bd[j] = FLT_MAX; bi[j] = -1; }
  }
}

/* ------------------------------------------------------------------------------------------ */
/* std::priority_queue<std::pair<float, tableint>, vector, CompareByFirst> restated            */
/* (include/hnswlib/hnswalg.h:71-76; heap moves = libstdc++ bits/stl_heap.h)                   */
/* ------------------------------------------------------------------------------------------ */
typedef struct { float d; uint32_t id; } ent_t;
typedef struct { ent_t *a; size_t n, cap; } pq_t;

static void pq_reserve(pq_t *h, size_t need) {
  if (need <= h->cap) return;
  size_t nc = h->cap ? h->cap * 2 : 256;
  while (nc < need) nc *= 2;
  h->a = (ent_t *)realloc(h->a, nc * sizeof(ent_t));
  h->cap = nc;
}
/* __push_heap: comp(parent, value) == parent.d < value.d */
static void heap_sift_up(ent_t *a, size_t hole, size_t top, ent_t v) {
  while (hole > top) {
    size_t parent = (hole - 1) / 2;
    if (!(a[parent].d < v.d)) break;
    a[hole] = a[parent];
    hole = parent;
  }
  a[hole] = v;
}
static void pq_push(pq_t *h, float d, uint32_t id) { /* emplace = push_back + push_heap */
  pq_reserve(h, h->n + 1);
  ent_t v = {d, id};
  h->n++;
  heap_sift_up(h->a, h->n - 1, 0, v);
}
static void pq_pop(pq_t *h) { /* pop_heap + pop_back: __pop_heap -> __adjust_heap */
  if (h->n > 1) {
    size_t len = h->n - 1;
    ent_t v = h->a[len];
    h->a[len] = h->a[0];
    size_t hole = 0, child = 0;
    while (child < (len - 1) / 2) {
      child = 2 * (child + 1);
      if (h->a[child].d < h->a[child - 1].d) child--;
      h->a[hole] = h->a[child];
      hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
      child = 2 * (child + 1);
      h->a[hole] = h->a[child - 1];
      hole = child - 1;
    }
    heap_sift_up(h->a, hole, 0, v);
  }
  h->n--;
}

/* ------------------------------------------------------------------------------------------ */
/* Graph view over the reference's own memory layout (hnswalg.h:45-49, :66, :708-736;          */
/* bindings/hnsw_bindings.cpp:549-671).                                                        */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
  const uint8_t *level0;       /* cur_element_count * size_data_per_element bytes             */
  size_t size_per_elem;        /* 4 + 4*maxM0 + M*code_bytes + 8                              */
  size_t offset_data;          /* 4 + 4*maxM0                                                 */
  size_t label_offset;         /* offset_data + M*code_bytes                                  */
  const uint8_t *links;        /* concatenated upper-level lists                              */
  const uint64_t *link_off;    /* per element byte offset into links                          */
  const int32_t *levels;       /* element_levels_                                             */
  size_t size_links_per_elem;  /* 4 + 4*maxM                                                  */
  int64_t n;
  int32_t maxlevel;
  uint32_t enterpoint;
  int M, Ks, code_bytes;
} graph_t;

static inline const uint8_t *g_rec0(const graph_t *g, uint32_t id) { return g->level0 + (size_t)id * g->size_per_elem; }
static inline const uint8_t *g_code(const graph_t *g, uint32_t id) { return g_rec0(g, id) + g->offset_data; }
static inline uint64_t g_label(const graph_t *g, uint32_t id) { uint64_t l; memcpy(&l, g_rec0(g, id) + g->label_offset, 8); return l; }
static inline int g_deleted(const graph_t *g, uint32_t id) { return g_rec0(g, id)[2] & 1; }        /* hnswalg.h:941-944 */
static inline unsigned g_count(const uint8_t *ll) { uint16_t c; memcpy(&c, ll, 2); return c; }     /* hnswalg.h:946-948 */
static inline const uint8_t *g_list(const graph_t *g, uint32_t id, int level) {                    /* hnswalg.h:486-496 */
  return level == 0 ? g_rec0(g, id) : g->links + g->link_off[id] + (size_t)(level - 1) * g->size_links_per_elem;
}
static inline uint32_t g_link(const uint8_t *ll, unsigned j) { uint32_t v; memcpy(&v, ll + 4 + 4 * j, 4); return v; }

typedef struct { pq_t top, cand; uint32_t *visited; uint32_t tag; } ws_t;

/* hnswalg.h:243-329 searchBaseLayerST<has_deletions, true>  (filter == NULL)
 * hnswalg.h:332-440 searchBaseLayerSTWithFilter             (filter != NULL: bit per internal id, set by
 * the Python wrapper for every node whose *label* is in the caller's list; the
 * reference tests binary_fuse16_contain(label), an approximate set with ~2^-16 false positives;
 * the exact bitmap is what that filter approximates -- SURVEY.md section 2 row 6). */
/* Test aid: where an exact fp32 tie leaves the reference's outcome to heap order, the GPU walk (which
 * keeps arrival order among equal keys) is free to differ; tests ask for the per-query count of such
 * events so that they can tell "differs at a tie" from "differs".  Two events are counted:
 *  - an entry is evicted from top_candidates while an equal key stays behind as the new lowerBound
 *    (the evicted node is still expanded by the reference because its distance is not > lowerBound);
 *  - two candidates with equal distance are next to each other at the top of candidate_set. */
static int64_t *g_tie_sink = 0;
ORC_API void orc_set_tie_sink(int64_t *sink) { g_tie_sink = sink; }

static void search_base(const graph_t *g, const float *table, uint32_t ep, size_t ef, int has_del,
                        const uint8_t *filter, ws_t *w, int64_t *hops, int64_t *nbrs, int64_t *evals,
                        int64_t *ties) {
  w->top.n = w->cand.n = 0;
  w->tag++;
  float lower;
  int ep_ok = filter ? (int)((filter[ep >> 3] >> (ep & 7)) & 1) : (!has_del || !g_deleted(g, ep));
  if (ep_ok) {
    float d = pq_lookup(table, g->M, g->Ks, g_code(g, ep), g->code_bytes);
    (*evals)++;
    lower = d;
    pq_push(&w->top, d, ep);
    pq_push(&w->cand, -d, ep);
  } else {
    lower = FLT_MAX;
    pq_push(&w->cand, -lower, ep);
  }
  w->visited[ep] = w->tag;
  while (w->cand.n) {
    ent_t cur = w->cand.a[0];
    if (filter) { if ((-cur.d) > lower) break; }                                   /* :371 */
    else if ((-cur.d) > lower && (w->top.n == ef || !has_del)) break;              /* :270 */
    pq_pop(&w->cand);
    if (ties && w->cand.n && w->cand.a[0].d == cur.d) (*ties)++;
    const uint8_t *ll = g_list(g, cur.id, 0);
    unsigned size = g_count(ll);
    (*hops)++;
    (*nbrs) += size;                                                               /* :279-282 */
    for (unsigned j = 0; j < size; j++) {
      uint32_t cid = g_link(ll, j);
      if (w->visited[cid] == w->tag) continue;
      w->visited[cid] = w->tag;
      float d = pq_lookup(table, g->M, g->Ks, g_code(g, cid), g->code_bytes);
      (*evals)++;
      if (w->top.n < ef || lower > d) {
        pq_push(&w->cand, -d, cid);
        int admit;
        if (filter) admit = (filter[cid >> 3] >> (cid & 7)) & 1;                                /* :423-426 */
        else admit = !has_del || !g_deleted(g, cid);                                            /* :314 */
        if (admit) pq_push(&w->top, d, cid);
        if (w->top.n > ef) {
          float gone = w->top.a[0].d;
          pq_pop(&w->top);
          if (ties && w->top.n && w->top.a[0].d == gone) (*ties)++;
        }
        if (w->top.n) lower = w->top.a[0].d;
      }
    }
  }
}

typedef struct { float d; uint64_t l; } res_t;
static int res_cmp(const void *a, const void *b) {
  const res_t *x = (const res_t *)a, *y = (const res_t *)b;
  if (x->d < y->d) return -1;
  if (x->d > y->d) return 1;
  return x->l < y->l ? -1 : (x->l > y->l);
}

/* hnswalg.h:1237-1295 searchKnn / :1297-1361 searchKnnWithFilter, then the unload loop of
 * bindings/hnsw_bindings.cpp:340-351 (priority_queue<pair<float,label>> popped farthest first
 * => rows ascending by (dist, label)).  Returns the number of results found per query in
 * `found`; the binding throws when found != k (:342-345).                                      */
ORC_API int orc_hnsw_search(const uint8_t *level0, uint64_t size_per_elem, uint64_t offset_data,
                            uint64_t label_offset, const uint8_t *links, const uint64_t *link_off,
                            const int32_t *levels, uint64_t size_links_per_elem, int64_t n,
                            int32_t maxlevel, uint32_t enterpoint, int M, int Ks, int code_bytes,
                            const float *tables, int64_t B, int k, int ef_, const uint8_t *filter,
                            uint64_t *out_labels, float *out_dists, int32_t *found,
                            int64_t *out_hops, int64_t *out_nbrs, int64_t *out_evals) {
  graph_t g = {level0, size_per_elem, offset_data, label_offset, links, link_off, levels,
               size_links_per_elem, n, maxlevel, enterpoint, M, Ks, code_bytes};
  if (n == 0) { for (int64_t b = 0; b < B; b++) found[b] = 0; return 0; }
  ws_t w;
  memset(&w, 0, sizeof(w));
  w.visited = (uint32_t *)calloc((size_t)n, sizeof(uint32_t));
  /* num_deleted_ (hnswalg.h:838-841) selects the deletion-aware instantiation in searchKnn (:1277);
   * searchKnnWithFilter tests has_deletions_ (:1343), which is never set true -- both filter
   * instantiations behave identically anyway (template args unused in :332-440). */
  int has_del = 0;
  for (int64_t i = 0; i < n && !has_del; i++) has_del = g_deleted(&g, (uint32_t)i);
  size_t ef = (size_t)(ef_ > k ? ef_ : k);
  res_t *res = (res_t *)malloc(sizeof(res_t) * (ef + 1));
  for (int64_t b = 0; b < B; b++) {
    const float *t = tables + (size_t)b * M * Ks;
    int64_t hops = 0, nbrs = 0, evals = 0;
    uint32_t cur = enterpoint;
    float curdist = pq_lookup(t, M, Ks, g_code(&g, cur), code_bytes);
    evals++;
    for (int level = maxlevel; level > 0; level--) {                               /* :1248-1274 */
      int changed = 1;
      while (changed) {
        changed = 0;
        const uint8_t *ll = g_list(&g, cur, level);
        unsigned size = g_count(ll);
        hops++;
        nbrs += size;
        for (unsigned i = 0; i < size; i++) {
          uint32_t cand = g_link(ll, i);
          float d = pq_lookup(t, M, Ks, g_code(&g, cand), code_bytes);
          evals++;
          if (d < curdist) { curdist = d; cur = cand; changed = 1; }
        }
      }
    }
    int64_t ties = 0;
    search_base(&g, t, cur, ef, has_del, filter, &w, &hops, &nbrs, &evals, g_tie_sink ? &ties : 0);
    while (w.top.n > (size_t)k) {                                                  /* :1286-1288 */
      float gone = w.top.a[0].d;
      pq_pop(&w.top);
      if (g_tie_sink && w.top.n && w.top.a[0].d == gone) ties++;    /* a tie at the k-th place */
    }
    int cnt = (int)w.top.n;
    for (int i = 0; i < cnt; i++) { res[i].d = w.top.a[i].d; res[i].l = g_label(&g, w.top.a[i].id); }
    qsort(res, (size_t)cnt, sizeof(res_t), res_cmp);
    for (int i = 0; i < k; i++) {
      out_dists[(size_t)b * k + i] = i < cnt ? res[i].d : FLT_MAX;
      out_labels[(size_t)b * k + i] = i < cnt ? res[i].l : UINT64_MAX;
    }
    found[b] = cnt;
    if (g_tie_sink) g_tie_sink[b] = ties;
    if (out_hops) out_hops[b] = hops;
    if (out_nbrs) out_nbrs[b] = nbrs;
    if (out_evals) out_evals[b] = evals;
  }
  free(res);
  free(w.visited);
  free(w.top.a);
  free(w.cand.a);
  return 0;
}

/* annlite/core/codec/pq.py:158-177 -> scipy.cluster.vq.vq (third-party; scipy, unpinned in
 * requirements.txt; container has scipy 1.18): nearest codeword per subspace under Euclidean
 * distance, first minimum wins.  scipy's kernel (cluster/_vq.pyx) evaluates fp32 inputs through
 * a BLAS expansion |x|^2 - 2x.c + |c|^2 when ds >= 5 and a naive loop otherwise, so its rounding
 * is BLAS-dependent and cannot be restated bit-exactly; this restatement is the mathematically
 * defined argmin (float64 accumulation, first minimum), and parity for `encode` is reported as a
 * mismatch RATE against scipy on near-ties only (SURVEY.md 8f rank 1: "parity unpinned"). */
ORC_API void orc_encode(const float *x, const float *cb, int64_t N, int M, int Ks, int ds, int code_bytes,
                        void *out) {
  const int D = M * ds;
  for (int64_t n = 0; n < N; n++)
    for (int m = 0; m < M; m++) {
      const float *v = x + (size_t)n * D + (size_t)m * ds;
      double best = 0;
      uint32_t arg = 0;
      for (int c = 0; c < Ks; c++) {
        const float *w = cb + ((size_t)m * Ks + c) * ds;
        double acc = 0;
        for (int j = 0; j < ds; j++) { double t = (double)v[j] - (double)w[j]; acc += t * t; }
        if (c == 0 || acc < best) { best = acc; arg = (uint32_t)c; }
      }
      size_t o = (size_t)n * M + m;
      if (code_bytes == 1) ((uint8_t *)out)[o] = (uint8_t)arg;
      else if (code_bytes == 2) ((uint16_t *)out)[o] = (uint16_t)arg;
      else ((uint32_t *)out)[o] = arg;
    }
}

/* ---------------------------------------------------------------------------------------------------
 * NOT the reference's algorithm: a scalar model of the product's single-list walk (hnsw_walk_fast in
 * annlite_b200/csrc/hnsw_search.cu -- one sorted list of at most ef (distance, node, expanded) entries,
 * no visited set, no candidate heap, arrival order among equal keys).  CPU tests run it beside
 * orc_hnsw_search to check the equivalence argument of DESIGN.md section 4 at sizes where a Python model
 * is too slow, including which rows an exact fp32 tie may change.  Pinned to the kernel by the capture in
 * tests/golden/b200_capture_c5_ef256.npz: it reproduces the kernel's result sets and hop counts row for row.
 * Same arguments as orc_hnsw_search without filter; rows come back ascending by (dist, label).        */
ORC_API int orc_single_list_walk(const uint8_t *level0, uint64_t size_per_elem, uint64_t offset_data,
                                 uint64_t label_offset, const uint8_t *links, const uint64_t *link_off,
                                 const int32_t *levels, uint64_t size_links_per_elem, int64_t n,
                                 int32_t maxlevel, uint32_t enterpoint, int M, int Ks, int code_bytes,
                                 const float *tables, int64_t B, int k, int ef_, uint64_t *out_labels,
                                 float *out_dists, int32_t *found, int64_t *out_hops, int64_t *out_nbrs) {
  graph_t g = {level0, size_per_elem, offset_data, label_offset, links, link_off, levels,
               size_links_per_elem, n, maxlevel, enterpoint, M, Ks, code_bytes};
  if (n == 0) { for (int64_t b = 0; b < B; b++) found[b] = 0; return 0; }
  const int ef = ef_ > k ? ef_ : k;
  float *K = (float *)malloc(sizeof(float) * (size_t)(ef + 1));
  uint32_t *V = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(ef + 1));
  uint8_t *X = (uint8_t *)malloc((size_t)(ef + 1));
  res_t *res = (res_t *)malloc(sizeof(res_t) * (size_t)(ef + 1));
  for (int64_t b = 0; b < B; b++) {
    const float *t = tables + (size_t)b * M * Ks;
    int64_t hops = 0, nbrs = 0;
    uint32_t cur = enterpoint;
    float curdist = pq_lookup(t, M, Ks, g_code(&g, cur), code_bytes);
    for (int level = maxlevel; level > 0; level--) {
      int changed = 1;
      while (changed) {
        changed = 0;
        const uint8_t *ll = g_list(&g, cur, level);
        unsigned size = g_count(ll);
        hops++;
        nbrs += size;
        for (unsigned i = 0; i < size; i++) {
          uint32_t cand = g_link(ll, i);
          float d = pq_lookup(t, M, Ks, g_code(&g, cand), code_bytes);
          if (d < curdist) { curdist = d; cur = cand; changed = 1; }
        }
      }
    }
    int size = 1;
    K[0] = curdist; V[0] = cur; X[0] = 1;
    uint32_t node = cur;
    for (;;) {
      const uint8_t *ll = g_list(&g, node, 0);
      unsigned cnt = g_count(ll);
      hops++;
      nbrs += cnt;
      const float worst = size >= ef ? K[ef - 1] : HUGE_VALF;     /* lowerBound as of the hop's start */
      for (unsigned j = 0; j < cnt; j++) {
        uint32_t x = g_link(ll, j);
        float d = pq_lookup(t, M, Ks, g_code(&g, x), code_bytes);
        if (!(d < worst)) continue;
        int pos = 0, dup = 0;
        while (pos < size && K[pos] <= d) pos++;                  /* after its equals */
        for (int i = pos - 1; i >= 0 && K[i] == d; i--) if (V[i] == x) { dup = 1; break; }
        if (dup || pos >= ef) continue;
        int ns = size < ef ? size + 1 : ef;
        memmove(K + pos + 1, K + pos, sizeof(float) * (size_t)(ns - 1 - pos));
        memmove(V + pos + 1, V + pos, sizeof(uint32_t) * (size_t)(ns - 1 - pos));
        memmove(X + pos + 1, X + pos, (size_t)(ns - 1 - pos));
        K[pos] = d; V[pos] = x; X[pos] = 0;
        size = ns;
      }
      int nx = -1;
      for (int i = 0; i < size; i++) if (!X[i]) { nx = i; break; }
      if (nx < 0) break;
      X[nx] = 1;
      node = V[nx];
    }
    int cnt = size < k ? size : k;
    for (int i = 0; i < cnt; i++) { res[i].d = K[i]; res[i].l = g_label(&g, V[i]); }
    qsort(res, (size_t)cnt, sizeof(res_t), res_cmp);
    for (int i = 0; i < k; i++) {
      out_dists[(size_t)b * k + i] = i < cnt ? res[i].d : FLT_MAX;
      out_labels[(size_t)b * k + i] = i < cnt ? res[i].l : UINT64_MAX;
    }
    found[b] = cnt;
    if (out_hops) out_hops[b] = hops;
    if (out_nbrs) out_nbrs[b] = nbrs;
  }
  free(K); free(V); free(X); free(res);
  return 0;
}

/* NOT the reference's algorithm either: the scalar model of hnsw_walk_flagged (one sorted list of every
 * candidate with a PASS flag, lowerBound read off the list, capacity `cap`; see hnsw_search.cu).  `filter`
 * is the internal-id bitmap of orc_hnsw_search or NULL (then deleted nodes do not pass).  found[b] = -1
 * when the list would outgrow `cap` (the kernel flags the query and the host re-runs the batch on the
 * bitmap walk); out_peak[b] = the largest list size reached (drives the host's capacity rule).          */
ORC_API int orc_flagged_walk(const uint8_t *level0, uint64_t size_per_elem, uint64_t offset_data,
                             uint64_t label_offset, const uint8_t *links, const uint64_t *link_off,
                             const int32_t *levels, uint64_t size_links_per_elem, int64_t n,
                             int32_t maxlevel, uint32_t enterpoint, int M, int Ks, int code_bytes,
                             const float *tables, int64_t B, int k, int ef_, const uint8_t *filter, int cap,
                             uint64_t *out_labels, float *out_dists, int32_t *found, int64_t *out_hops,
                             int64_t *out_nbrs, int32_t *out_peak) {
  graph_t g = {level0, size_per_elem, offset_data, label_offset, links, link_off, levels,
               size_links_per_elem, n, maxlevel, enterpoint, M, Ks, code_bytes};
  if (n == 0) { for (int64_t b = 0; b < B; b++) found[b] = 0; return 0; }
  const int ef = ef_ > k ? ef_ : k;
  int has_del = 0;
  for (int64_t i = 0; i < n && !has_del; i++) has_del = g_deleted(&g, (uint32_t)i);
  const size_t room = (size_t)cap + 65;
  float *K = (float *)malloc(sizeof(float) * room);
  uint32_t *V = (uint32_t *)malloc(sizeof(uint32_t) * room);
  uint8_t *X = (uint8_t *)malloc(room), *P = (uint8_t *)malloc(room);
  res_t *res = (res_t *)malloc(sizeof(res_t) * room);
  for (int64_t b = 0; b < B; b++) {
    const float *t = tables + (size_t)b * M * Ks;
    int64_t hops = 0, nbrs = 0;
    uint32_t cur = enterpoint;
    float curdist = pq_lookup(t, M, Ks, g_code(&g, cur), code_bytes);
    for (int level = maxlevel; level > 0; level--) {
      int changed = 1;
      while (changed) {
        changed = 0;
        const uint8_t *ll = g_list(&g, cur, level);
        unsigned size = g_count(ll);
        hops++;
        nbrs += size;
        for (unsigned i = 0; i < size; i++) {
          uint32_t cand = g_link(ll, i);
          float d = pq_lookup(t, M, Ks, g_code(&g, cand), code_bytes);
          if (d < curdist) { curdist = d; cur = cand; changed = 1; }
        }
      }
    }
#define PASSES(id) (filter ? (int)((filter[(id) >> 3] >> ((id) & 7)) & 1) : !g_deleted(&g, (id)))
    int size = 1, peak = 1, aborted = 0;
    K[0] = curdist; V[0] = cur; X[0] = 1; P[0] = (uint8_t)PASSES(cur);
    int npass = P[0];
    float lb = P[0] ? curdist : FLT_MAX;
    uint32_t node = cur;
    for (;;) {
      const uint8_t *ll = g_list(&g, node, 0);
      unsigned cnt = g_count(ll);
      hops++;
      nbrs += cnt;
      const float lb0 = lb;
      const int npass0 = npass, size0 = size;
      int added = 0;
      for (unsigned j = 0; j < cnt; j++) {
        uint32_t x = g_link(ll, j);
        float d = pq_lookup(t, M, Ks, g_code(&g, x), code_bytes);
        if (!(npass0 < ef || d < lb0)) continue;                 /* :306 / :413 at the hop's start */
        int pos = 0, dup = 0;
        while (pos < size && K[pos] <= d) pos++;
        for (int i = pos - 1; i >= 0 && K[i] == d; i--) if (V[i] == x) { dup = 1; break; }
        if (dup) continue;
        if (size0 + ++added > cap) { aborted = 1; break; }
        memmove(K + pos + 1, K + pos, sizeof(float) * (size_t)(size - pos));
        memmove(V + pos + 1, V + pos, sizeof(uint32_t) * (size_t)(size - pos));
        memmove(X + pos + 1, X + pos, (size_t)(size - pos));
        memmove(P + pos + 1, P + pos, (size_t)(size - pos));
        K[pos] = d; V[pos] = x; X[pos] = 0; P[pos] = (uint8_t)PASSES(x);
        size++;
      }
      if (aborted) break;
      if (size > peak) peak = size;
      if (added) {
        int total = 0, pef = -1, plast = -1;
        for (int i = 0; i < size; i++) if (P[i]) { total++; plast = i; if (total == ef && pef < 0) pef = i; }
        if (total >= ef) { size = pef + 1; npass = ef; lb = K[pef]; }
        else { npass = total; if (total > 0) lb = K[plast]; }
      }
      int nx = -1;
      for (int i = 0; i < size; i++) if (!X[i]) { nx = i; break; }
      if (nx < 0) break;
      if (filter) { if (K[nx] > lb) break; }
      else if (K[nx] > lb && (npass == ef || !has_del)) break;
      X[nx] = 1;
      node = V[nx];
    }
#undef PASSES
    int cnt = 0;
    if (!aborted)
      for (int i = 0; i < size && cnt < k; i++) if (P[i]) { res[cnt].d = K[i]; res[cnt].l = g_label(&g, V[i]); cnt++; }
    qsort(res, (size_t)cnt, sizeof(res_t), res_cmp);
    for (int i = 0; i < k; i++) {
      out_dists[(size_t)b * k + i] = i < cnt ? res[i].d : FLT_MAX;
      out_labels[(size_t)b * k + i] = i < cnt ? res[i].l : UINT64_MAX;
    }
    found[b] = aborted ? -1 : cnt;
    if (out_hops) out_hops[b] = hops;
    if (out_nbrs) out_nbrs[b] = nbrs;
    if (out_peak) out_peak[b] = peak;
  }
  free(K); free(V); free(X); free(P); free(res);
  return 0;
}

/* NOT the reference's algorithm either: the scalar model of hnsw_walk4f (annlite_b200/csrc/walk_flagged4.cu), the
 * filtered / deletion-aware walk on TWO sorted lists -- P = admitted entries (top_candidates, at most ef), N =
 * traversed-but-not-admitted entries (candidate_set minus top_candidates, capacity cap_n) -- with the kernel's order of
 * operations: the smallest new candidate of a hop is compared with the nearest unexpanded entry first (that decides
 * the next node), the others follow in neighbour order; lowerBound is P's ef-th key once P is full, else P's largest
 * key, else FLT_MAX; N keeps its cap_n smallest entries, and an entry that falls off its end only matters (found =
 * -1: the host re-runs the query on the bitmap walk) if it could still have been expanded (P not full, or its key
 * <= lowerBound).  out_peak_n = the largest number of N entries that could still be expanded.                       */
typedef struct { float k; uint32_t v; uint8_t x; } tl_ent;
static int tl_listed(const tl_ent *a, int n, uint32_t id) { for (int i = 0; i < n; i++) if (a[i].v == id) return 1; return 0; }
static void tl_insert(tl_ent *a, int *n, float key, uint32_t id, int expanded) {
  int pos = 0;
  while (pos < *n && a[pos].k <= key) pos++;                          /* after its equals: arrival order */
  memmove(a + pos + 1, a + pos, sizeof(tl_ent) * (size_t)(*n - pos));
  a[pos].k = key; a[pos].v = id; a[pos].x = (uint8_t)expanded;
  (*n)++;
}
ORC_API int orc_two_list_walk(const uint8_t *level0, uint64_t size_per_elem, uint64_t offset_data,
                              uint64_t label_offset, const uint8_t *links, const uint64_t *link_off,
                              const int32_t *levels, uint64_t size_links_per_elem, int64_t n,
                              int32_t maxlevel, uint32_t enterpoint, int M, int Ks, int code_bytes,
                              const float *tables, int64_t B, int k, int ef_, const uint8_t *filter, int cap_n,
                              uint64_t *out_labels, float *out_dists, int32_t *found, int64_t *out_hops,
                              int64_t *out_nbrs, int32_t *out_peak_n) {
  graph_t g = {level0, size_per_elem, offset_data, label_offset, links, link_off, levels,
               size_links_per_elem, n, maxlevel, enterpoint, M, Ks, code_bytes};
  if (n == 0) { for (int64_t b = 0; b < B; b++) found[b] = 0; return 0; }
  const int ef = ef_ > k ? ef_ : k;
  int has_del = 0;
  for (int64_t i = 0; i < n && !has_del; i++) has_del = g_deleted(&g, (uint32_t)i);
  const int size_guard = !filter && has_del;
  tl_ent *P = (tl_ent *)malloc(sizeof(tl_ent) * (size_t)(ef + 80));
  tl_ent *N = (tl_ent *)malloc(sizeof(tl_ent) * (size_t)(cap_n + 2));
  res_t *res = (res_t *)malloc(sizeof(res_t) * (size_t)(ef + 1));
  for (int64_t b = 0; b < B; b++) {
    const float *t = tables + (size_t)b * M * Ks;
    int64_t hops = 0, nbrs = 0;
    uint32_t cur = enterpoint;
    float curdist = pq_lookup(t, M, Ks, g_code(&g, cur), code_bytes);
    for (int level = maxlevel; level > 0; level--) {
      int changed = 1;
      while (changed) {
        changed = 0;
        const uint8_t *ll = g_list(&g, cur, level);
        unsigned size = g_count(ll);
        hops++;
        nbrs += size;
        for (unsigned i = 0; i < size; i++) {
          uint32_t cand = g_link(ll, i);
          float d = pq_lookup(t, M, Ks, g_code(&g, cand), code_bytes);
          if (d < curdist) { curdist = d; cur = cand; changed = 1; }
        }
      }
    }
#define TL_PASSES(id) (filter ? (int)((filter[(id) >> 3] >> ((id) & 7)) & 1) : !g_deleted(&g, (id)))
    int sp = 0, sn = 0, aborted = 0, peak = 0;
    const int ep_pass = TL_PASSES(cur);
    if (ep_pass) tl_insert(P, &sp, curdist, cur, 1); else tl_insert(N, &sn, curdist, cur, 1);
    float lb = ep_pass ? curdist : FLT_MAX, pmax = ep_pass ? curdist : -HUGE_VALF;
    int have_lost = 0; float lost = 0.f;
    uint32_t node = cur;
    for (;;) {
      const uint8_t *ll = g_list(&g, node, 0);
      unsigned cnt = g_count(ll);
      hops++;
      nbrs += cnt;
      const int admit_all = sp < ef;
      const float worst = lb;
      float ck[64]; uint32_t cid[64]; uint8_t cp[64], live[64];
      for (unsigned j = 0; j < cnt; j++) {
        cid[j] = g_link(ll, j);
        ck[j] = pq_lookup(t, M, Ks, g_code(&g, cid[j]), code_bytes);
        cp[j] = (uint8_t)TL_PASSES(cid[j]);
        live[j] = (uint8_t)(admit_all || ck[j] < worst);               /* :306 / :413 at the hop's start */
      }
      /* nearest unexpanded entry of either list (P before N among equal keys) */
      int e2l = -1, e2i = -1; float e2k = 0.f;
      for (int i = 0; i < sp; i++) if (!P[i].x) { e2l = 0; e2i = i; e2k = P[i].k; break; }
      for (int i = 0; i < sn; i++) if (!N[i].x) { if (e2l < 0 || N[i].k < e2k) { e2l = 1; e2i = i; e2k = N[i].k; } break; }
      /* phase A: smallest new candidate (lower j among equals) that is not listed */
      int have_new = 0, src = -1;
      for (;;) {
        src = -1;
        for (unsigned j = 0; j < cnt; j++) if (live[j] && (src < 0 || ck[j] < ck[src])) src = (int)j;
        if (src < 0) break;
        live[src] = 0;
        if (!tl_listed(P, sp, cid[src]) && !tl_listed(N, sn, cid[src])) { have_new = 1; break; }
      }
#define TL_INSERT(key, id, pass, expd)                                                            \
  do {                                                                                            \
    if (pass) { tl_insert(P, &sp, (key), (id), (expd)); if ((key) > pmax) pmax = (key);           \
                if (sp > ef + 64) sp = ef + 64; }                                                 \
    else {                                                                                        \
      if (sn == cap_n) {                                                                          \
        float lastk = N[sn - 1].k, m_ = lastk > (key) ? lastk : (key);                            \
        if (!have_lost || m_ < lost) { lost = m_; have_lost = 1; }                                \
      }                                                                                           \
      tl_insert(N, &sn, (key), (id), (expd));                                                     \
      if (sn > cap_n) sn = cap_n;                                                                 \
    }                                                                                             \
  } while (0)
      float nextkey; uint32_t next;
      if (have_new && (e2l < 0 || ck[src] < e2k)) {
        next = cid[src]; nextkey = ck[src];
        TL_INSERT(ck[src], cid[src], cp[src], 1);
      } else {
        if (e2l < 0) break;                                              /* candidate_set exhausted */
        if (e2l == 0) { P[e2i].x = 1; next = P[e2i].v; } else { N[e2i].x = 1; next = N[e2i].v; }
        nextkey = e2k;
        if (have_new) TL_INSERT(ck[src], cid[src], cp[src], 0);
      }
      if (have_new) {
        for (unsigned j = 0; j < cnt; j++) {
          if (!live[j]) continue;
          if (tl_listed(P, sp, cid[j]) || tl_listed(N, sn, cid[j])) continue;
          TL_INSERT(ck[j], cid[j], cp[j], 0);
        }
        if (sp >= ef) {
          sp = ef;
          lb = P[ef - 1].k;   /* N is NOT pruned: entries beyond lowerBound are never expanded (break rule below) and are
                                 the first to fall off N's end when it is full -- harmless, see `lost` */
        } else if (sp > 0) lb = pmax;
        { int need = 0;       /* the capacity this query needs: N entries that may still be expanded */
          for (int i = 0; i < sn; i++) need += (sp < ef) || !(N[i].k > lb);
          if (need > peak) peak = need; }
        if (have_lost && !(sp >= ef && lost > lb)) { aborted = 1; break; }
      }
      if (nextkey > lb && (!size_guard || sp >= ef)) break;              /* :371 / :270 */
      node = next;
    }
#undef TL_INSERT
#undef TL_PASSES
    int cnt = 0;
    if (!aborted) for (int i = 0; i < sp && i < ef && cnt < k; i++) { res[cnt].d = P[i].k; res[cnt].l = g_label(&g, P[i].v); cnt++; }
    qsort(res, (size_t)cnt, sizeof(res_t), res_cmp);
    for (int i = 0; i < k; i++) {
      out_dists[(size_t)b * k + i] = i < cnt ? res[i].d : FLT_MAX;
      out_labels[(size_t)b * k + i] = i < cnt ? res[i].l : UINT64_MAX;
    }
    found[b] = aborted ? -1 : cnt;
    if (out_hops) out_hops[b] = hops;
    if (out_nbrs) out_nbrs[b] = nbrs;
    if (out_peak_n) out_peak_n[b] = peak;
  }
  free(P); free(N); free(res);
  return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* NOT the reference: one batch of back-links of the product's batched GPU build             */
/* ------------------------------------------------------------------------------------------ */

/* The back-link step of oracle/gpu_build_model.py (whose numpy form, backlinks_numpy, is this function's
 * CPU-side reference).  Rows i = 0..B-1 of a batch became nodes x = first + i; row i links back to its
 * min(found[i], k) candidates r = sel[i*k + j] at distance dist[i*k + j], in pair order p = i*k + j.  A
 * neighbour with room appends x; a full one becomes [x] + those of its neighbours c with !(D(x, c) < d),
 * in descending id, at most maxM0 in all: hnswalg.h:575-616 in PQ mode (hnsw_build.cpp connect()), where
 * D(x, c) = PQLookup of c's code in x's table.  queue_order = 0 stores that list in descending id, as the
 * GPU builder does; 1 stores it in the order the reference's queue gives it back: every kept entry has the
 * same key d, so that is the pop order of a max-heap of equal keys pushed in descending id (heap_pop_order).
 * Slots past a rewritten list's count keep their old bytes, as the host builder leaves them.  level0: host-layout records (count u16 at 0, links u32 from byte 4,
 * u8 codes at offset_data).  counts[0..2] += appends, rewrites, rewrites that dropped a neighbour. */
/* The order in which std::priority_queue (libstdc++ std::pop_heap / __adjust_heap) gives back n entries of
 * EQUAL key pushed as 0..n-1: push_heap moves nothing, and each pop takes the front and sifts the last entry in
 * along the right children.  out[s] = the push position of the s-th entry popped. */
static void heap_pop_order(int n, int *out) {
  int a[2048];
  for (int i = 0; i < n; i++) a[i] = i;
  for (int s = 0, len = n; len > 0; s++, len--) {
    out[s] = a[0];
    const int L = len - 1, val = a[L];
    int hole = 0, child = 0;
    while (child < (L - 1) / 2) {
      child = 2 * (child + 1);
      a[hole] = a[child];
      hole = child;
    }
    if ((L & 1) == 0 && child == (L - 2) / 2) {
      child = 2 * (child + 1);
      a[hole] = a[child - 1];
      hole = child - 1;
    }
    if (L) a[hole] = val;
  }
}

ORC_API void orc_build_backlinks(uint8_t *level0, uint64_t size_per_elem, uint64_t offset_data, int maxM0, int M,
                                 int Ks, const float *tables, const uint64_t *sel, const float *dist,
                                 const int32_t *found, int64_t B, int k, uint32_t first, int queue_order,
                                 int64_t *counts) {
  uint32_t *keep = malloc((size_t)maxM0 * sizeof(uint32_t));
  int *order = malloc((size_t)maxM0 * sizeof(int));
  for (int64_t i = 0; i < B; i++) {
    const uint32_t x = first + (uint32_t)i;
    const float *T = tables + (size_t)i * M * Ks;
    const int nf = found[i] < k ? found[i] : k;
    for (int j = 0; j < nf; j++) {
      const uint32_t r = (uint32_t)sel[(size_t)i * k + j];
      const float dr = dist[(size_t)i * k + j];
      uint8_t *rec = level0 + (size_t)r * size_per_elem;
      uint16_t cnt;
      memcpy(&cnt, rec, 2);
      if (cnt < maxM0) {
        memcpy(rec + 4 + 4 * (size_t)cnt, &x, 4);
        cnt++;
        memcpy(rec, &cnt, 2);
        counts[0]++;
        continue;
      }
      int nk = 0;
      for (int s = 0; s < cnt; s++) {
        uint32_t c;
        memcpy(&c, rec + 4 + 4 * (size_t)s, 4);
        const uint8_t *code = level0 + (size_t)c * size_per_elem + offset_data;
        float d = 0.f;
        for (int m = 0; m < M; m++) d += T[(size_t)m * Ks + code[m]];
        if (!(d < dr)) {
          int t = nk++;
          while (t > 0 && keep[t - 1] < c) { keep[t] = keep[t - 1]; t--; }  /* descending id */
          keep[t] = c;
        }
      }
      const int total = 1 + nk < maxM0 ? 1 + nk : maxM0;
      if (queue_order) heap_pop_order(total, order);
      else for (int s = 0; s < total; s++) order[s] = s;
      for (int s = 0; s < total; s++) memcpy(rec + 4 + 4 * (size_t)s, order[s] ? &keep[order[s] - 1] : &x, 4);
      cnt = (uint16_t)total;
      memcpy(rec, &cnt, 2);
      counts[1]++;
      if (1 + nk > maxM0) counts[2]++;
    }
  }
  free(keep);
  free(order);
}
