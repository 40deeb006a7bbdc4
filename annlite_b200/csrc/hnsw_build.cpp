// hnsw_build.cpp -- host-side HNSW graph: storage in the reference's byte layout, the
// hnswlib-compatible save/load format, and multi-threaded insertion.
//
// Construction is the SURVEY.md section 8f "next" row 2: a host C++ implementation that follows
// the reference's insertion algorithm (include/hnswlib/hnswalg.h:1108-1235 addPoint, :158-238
// searchBaseLayer, :443-483 getNeighborsByHeuristic2, :502-619 mutuallyConnectNewElement) closely
// enough that a single-threaded build produces a byte-identical graph (tests/test_host_graph.py, tests/test_update_parity.py
// compares against a graph the compiled reference built from the same inputs).  That includes
// the reference's PQ-mode quirk (SURVEY.md section 0.2): PQLookup ignores its first argument, so
// every "distance between two stored nodes" is really the distance from the point being inserted
// to the second node.  Here that is explicit: all distances are dist_to_new(id).
//
// The per-point ADC table comes from the GPU (K1) in batches; this file only consumes tables.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <queue>
#include <random>
#include <sched.h>
#include <thread>
#include <unordered_set>

#include "annb_internal.h"

// ------------------------------------------------------------------------------------------------
// HostGraph storage
// ------------------------------------------------------------------------------------------------
HostGraph::~HostGraph() { clear(); }

void HostGraph::clear() {
  if (level0) free(level0);
  level0 = nullptr;
  for (auto p : upper)
    if (p) free(p);
  upper.clear();
  levels.clear();
  label_lookup.clear();
  count = 0;
  maxlevel = -1;
  enterpoint = 0xFFFFFFFFu;
  num_deleted = 0;
  inited = false;
}

uint64_t HostGraph::label(uint32_t id) const {
  uint64_t l;
  memcpy(&l, rec0(id) + label_offset, 8);
  return l;
}

// HierarchicalNSW(space, max_elements, M, ef_construction, seed): hnswalg.h:27-69
int HostGraph::init(int64_t max_elems, int M_, int efc, uint64_t seed_, size_t code_row_bytes_) {
  clear();
  M = M_;
  maxM = M_;
  maxM0 = 2 * M_;
  ef_construction = std::max(efc, M_);
  seed = seed_;
  code_row_bytes = code_row_bytes_;
  size_links_level0 = (size_t)maxM0 * 4 + 4;
  size_per_elem = size_links_level0 + code_row_bytes + 8;
  offset_data = size_links_level0;
  label_offset = size_links_level0 + code_row_bytes;
  size_links_per_elem = (size_t)maxM * 4 + 4;
  mult = 1.0 / std::log(1.0 * M);
  level_gen.seed((std::default_random_engine::result_type)seed_);  // hnswalg.h:42
  max_elements = max_elems;
  level0 = (uint8_t *)malloc(std::max<size_t>(1, (size_t)max_elems * size_per_elem));
  if (!level0) ANNB_FAIL(ANNB_ENOMEM, "Not enough memory");
  upper.assign((size_t)max_elems, nullptr);
  levels.assign((size_t)max_elems, 0);
  label_lookup.reserve((size_t)max_elems);  // no rehash under the insertion lock
  inited = true;
  return ANNB_OK;
}

// resizeIndex: hnswalg.h:680-706
int HostGraph::resize(int64_t new_max) {
  if (new_max < count.load()) ANNB_FAIL(ANNB_EINVAL, "Cannot resize, max element is less than the current number of elements");
  uint8_t *nl = (uint8_t *)realloc(level0, std::max<size_t>(1, (size_t)new_max * size_per_elem));
  if (!nl) ANNB_FAIL(ANNB_ENOMEM, "Not enough memory: resizeIndex failed to allocate base layer");
  level0 = nl;
  upper.resize((size_t)new_max, nullptr);
  levels.resize((size_t)new_max, 0);
  label_lookup.reserve((size_t)new_max);
  max_elements = new_max;
  return ANNB_OK;
}

// saveIndex: hnswalg.h:708-736
int HostGraph::save_file(const char *path) const {
  FILE *f = fopen(path, "wb");
  if (!f) ANNB_FAIL(ANNB_EIO, "Cannot open file");
  const uint64_t n = (uint64_t)count.load();
  uint64_t hdr6[6] = {0, (uint64_t)max_elements, n, (uint64_t)size_per_elem, (uint64_t)label_offset, (uint64_t)offset_data};
  fwrite(hdr6, 8, 6, f);
  fwrite(&maxlevel, 4, 1, f);
  fwrite(&enterpoint, 4, 1, f);
  uint64_t m3[3] = {(uint64_t)maxM, (uint64_t)maxM0, (uint64_t)M};
  fwrite(m3, 8, 3, f);
  fwrite(&mult, 8, 1, f);
  uint64_t efc = (uint64_t)ef_construction;
  fwrite(&efc, 8, 1, f);
  fwrite(level0, 1, n * size_per_elem, f);
  for (uint64_t i = 0; i < n; i++) {
    uint32_t sz = levels[i] > 0 ? (uint32_t)(size_links_per_elem * levels[i]) : 0;
    fwrite(&sz, 4, 1, f);
    if (sz) fwrite(upper[i], 1, sz, f);
  }
  bool ok = !ferror(f);
  fclose(f);
  if (!ok) ANNB_FAIL(ANNB_EIO, "write failed: %s", path);
  return ANNB_OK;
}

namespace {
constexpr uint64_t kMaxListLinks = 2048;  // maxM0 = 2*M <= 2048 (annb_init_graph limits M to 1024)
constexpr int kMaxLevels = 63;
}  // namespace

int HostGraph::validate() const {
  const int64_t n = count.load();
  if (n < 0 || n > max_elements) ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (element count)");
  if (n == 0) {  // the empty graph of hnswalg.h:61-62
    if (enterpoint != 0xFFFFFFFFu || maxlevel != -1)
      ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (empty graph with entry point %u, max level %d)", enterpoint, maxlevel);
    return ANNB_OK;
  }
  if (enterpoint >= (uint64_t)n || maxlevel < 0 || maxlevel >= kMaxLevels || levels[enterpoint] < maxlevel)
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (entry point %u, max level %d)", enterpoint, maxlevel);
  for (int64_t i = 0; i < n; i++) {
    const int lv = levels[i];
    if (lv < 0 || lv >= kMaxLevels || lv > maxlevel || (lv > 0 && !upper[i]))
      ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (level %d of node %lld)", lv, (long long)i);
    for (int l = 0; l <= lv; l++) {
      const uint8_t *ll = list_at((uint32_t)i, l);
      uint16_t c;
      memcpy(&c, ll, 2);
      if (c > (l ? maxM : maxM0))
        ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (%u links on level %d of node %lld)", c, l, (long long)i);
      for (unsigned j = 0; j < c; j++) {
        uint32_t t;
        memcpy(&t, ll + 4 + 4 * j, 4);
        if (t >= (uint64_t)n || levels[t] < l)
          ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (link %u on level %d of node %lld)", t, l, (long long)i);
      }
    }
  }
  return ANNB_OK;
}

// loadIndex: hnswalg.h:738-846
int HostGraph::load_file(const char *path, int64_t max_elements_i, size_t code_row_bytes_) {
  FILE *f = fopen(path, "rb");
  if (!f) ANNB_FAIL(ANNB_EIO, "Cannot open file");
  fseek(f, 0, SEEK_END);
  const long total = ftell(f);
  fseek(f, 0, SEEK_SET);
  uint64_t hdr6[6], m3[3], efc;
  int32_t ml;
  uint32_t ep;
  double mu;
  bool ok = fread(hdr6, 8, 6, f) == 6 && fread(&ml, 4, 1, f) == 1 && fread(&ep, 4, 1, f) == 1 &&
            fread(m3, 8, 3, f) == 3 && fread(&mu, 8, 1, f) == 1 && fread(&efc, 8, 1, f) == 1;
  if (!ok) {
    fclose(f);
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
  }
  const uint64_t n = hdr6[2];
  const size_t spe = hdr6[3];
  const size_t expect = (size_t)m3[1] * 4 + 4 + code_row_bytes_ + 8;
  if (m3[0] < 1 || m3[0] > kMaxListLinks || m3[1] < 1 || m3[1] > kMaxListLinks || m3[2] < 1 || m3[2] > kMaxListLinks) {
    fclose(f);
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (M=%llu, maxM=%llu, maxM0=%llu)",
              (unsigned long long)m3[2], (unsigned long long)m3[0], (unsigned long long)m3[1]);
  }
  if (spe != expect || hdr6[5] != m3[1] * 4 + 4 || hdr6[4] != m3[1] * 4 + 4 + code_row_bytes_) {
    fclose(f);
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported (element size %zu, expected %zu for this PQ geometry)", spe, expect);
  }
  // everything that sizes an allocation or a read is checked against the file before anything is allocated
  const uint64_t kMaxNodes = 0xfffffffeull;  // internal ids are 32-bit, 0xffffffff marks "no entry point"
  if (n > kMaxNodes || hdr6[1] > kMaxNodes || total < 96 || n > ((uint64_t)total - 96) / (spe + 4) || ml < -1 || ml >= kMaxLevels ||
      efc < 1 || efc > (1ull << 31) || !std::isfinite(mu) || mu < 0.0 || mu > 64.0) {
    fclose(f);
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
  }
  int64_t maxel = max_elements_i;
  if (maxel < (int64_t)n) maxel = (int64_t)hdr6[1];  // hnswalg.h:766-768
  if (maxel < (int64_t)n) maxel = (int64_t)n;        // a file whose own limit is below its count: keep what it holds
  if ((uint64_t)maxel > kMaxNodes) {
    fclose(f);
    ANNB_FAIL(ANNB_EINVAL, "max_elements exceeds the 32-bit internal id space");
  }
  clear();
  M = (int)m3[2];
  maxM = (int)m3[0];
  maxM0 = (int)m3[1];
  ef_construction = (int)efc;
  mult = mu;
  code_row_bytes = code_row_bytes_;
  size_links_level0 = (size_t)maxM0 * 4 + 4;
  size_per_elem = spe;
  offset_data = hdr6[5];
  label_offset = hdr6[4];
  size_links_per_elem = (size_t)maxM * 4 + 4;
  max_elements = maxel;
  maxlevel = ml;
  enterpoint = ep;
  level0 = (uint8_t *)malloc(std::max<size_t>(1, (size_t)maxel * spe));
  if (!level0) {
    fclose(f);
    ANNB_FAIL(ANNB_ENOMEM, "Not enough memory: loadIndex failed to allocate level0");
  }
  if (fread(level0, 1, n * spe, f) != n * spe) {
    fclose(f);
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
  }
  upper.assign((size_t)maxel, nullptr);
  levels.assign((size_t)maxel, 0);
  for (uint64_t i = 0; i < n; i++) {
    uint32_t sz;
    if (fread(&sz, 4, 1, f) != 1) {
      fclose(f);
      ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
    }
    if (sz) {
      const long here = ftell(f);
      if (sz % size_links_per_elem != 0 || sz / size_links_per_elem >= (size_t)kMaxLevels || here < 0 || (uint64_t)sz > (uint64_t)(total - here)) {
        fclose(f);
        ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
      }
      levels[i] = (int32_t)(sz / size_links_per_elem);
      upper[i] = (uint8_t *)malloc(sz);
      if (!upper[i] || fread(upper[i], 1, sz, f) != sz) {
        fclose(f);
        ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
      }
    }
  }
  if (ftell(f) != total) {
    fclose(f);
    ANNB_FAIL(ANNB_EIO, "Index seems to be corrupted or unsupported");
  }
  fclose(f);
  count = (int64_t)n;
  num_deleted = 0;
  if (int rc = validate()) {
    count = 0;
    return rc;
  }
  level_gen = std::default_random_engine();  // the loading constructor never seeds it (hnswalg.h:23-25)
  label_lookup.reserve(n);
  for (uint64_t i = 0; i < n; i++) {
    label_lookup[label((uint32_t)i)] = (uint32_t)i;
    if (deleted((uint32_t)i)) num_deleted++;
  }
  inited = true;
  return ANNB_OK;
}

// ------------------------------------------------------------------------------------------------
// insertion
// ------------------------------------------------------------------------------------------------
namespace {

using Near = std::pair<float, uint32_t>;
struct FartherFirst {  // CompareByFirst, hnswalg.h:71-76
  bool operator()(const Near &a, const Near &b) const noexcept { return a.first < b.first; }
};
// std::priority_queue is specified as push_back + std::push_heap / std::pop_heap + pop_back over its container;
// this wrapper is exactly that over a vector that is REUSED between calls (clear() keeps the capacity), so an
// insertion performs no heap allocations while its tie behaviour stays identical to the reference's queues.
template <class Cmp>
struct ReHeap {
  std::vector<Near> v;
  Cmp cmp;
  void clear() { v.clear(); }
  bool empty() const { return v.empty(); }
  size_t size() const { return v.size(); }
  const Near &top() const { return v.front(); }
  void emplace(float d, uint32_t id) {
    v.emplace_back(d, id);
    std::push_heap(v.begin(), v.end(), cmp);
  }
  void push(const Near &n) {
    v.push_back(n);
    std::push_heap(v.begin(), v.end(), cmp);
  }
  void pop() {
    std::pop_heap(v.begin(), v.end(), cmp);
    v.pop_back();
  }
};
using FarHeap = ReHeap<FartherFirst>;
constexpr unsigned kMaxLinks = 2048;  // maxM0 = 2*M <= 2048 (annb_init_graph limits M to 1024)

inline unsigned list_count(const uint8_t *ll) {
  uint16_t c;
  memcpy(&c, ll, 2);
  return c;
}
inline void set_list_count(uint8_t *ll, unsigned c) {
  uint16_t v = (uint16_t)c;
  memcpy(ll, &v, 2);
}
inline uint32_t *list_links(uint8_t *ll) { return reinterpret_cast<uint32_t *>(ll + 4); }

struct SpinLocks {
  std::unique_ptr<std::atomic<uint8_t>[]> f;
  size_t n = 0;
  void reset(size_t m) {
    f.reset(new std::atomic<uint8_t>[m]);
    for (size_t i = 0; i < m; i++) f[i].store(0, std::memory_order_relaxed);
    n = m;
  }
  void lock(size_t i) {
    // A node can stay locked for a whole insertion (~1 ms, see Worker::insert), so waiters back off:
    // a short busy phase, then yields, then sleeps -- 100+ inserting threads must not burn their
    // hyper-thread siblings' cycles while they wait.
    int spins = 0;
    for (;;) {
      uint8_t e = 0;
      if (f[i].compare_exchange_weak(e, 1, std::memory_order_acquire)) return;
      while (f[i].load(std::memory_order_relaxed)) {
        if (++spins < 64) {
#if defined(__x86_64__)
          __builtin_ia32_pause();
#endif
        } else if (spins < 96) {
          std::this_thread::yield();
        } else {
          std::this_thread::sleep_for(std::chrono::microseconds(20));
        }
      }
    }
  }
  void unlock(size_t i) { f[i].store(0, std::memory_order_release); }
};
struct SpinGuard {
  SpinLocks &l;
  size_t i;
  bool held;
  SpinGuard(SpinLocks &l_, size_t i_, bool take = true) : l(l_), i(i_), held(take) {
    if (take) l.lock(i);
  }
  ~SpinGuard() {
    if (held) l.unlock(i);
  }
};

struct SharedBuild {
  HostGraph *g;
  SpinLocks node_locks;
  std::mutex global, count_guard, rng_guard;
  std::default_random_engine *level_gen;  // hnswalg.h:130 (state lives in HostGraph)
  int n_sub, Ks, code_bytes;
  bool threaded;
};

struct Worker {
  SharedBuild &S;
  HostGraph &g;
  std::vector<uint16_t> seen;  // visited tags, 16-bit like vl_type (hnswlib/visited_list_pool.h:8-30)
  uint16_t tag = 0;
  FarHeap h_top, h_cand, h_cands, h_filtered;  // reused across insertions
  ReHeap<std::less<Near>> h_closest;
  std::vector<Near> kept;
  std::vector<uint32_t> sel;
  // device-graph patching: level-0 records this worker rewrote, and whether anything above level 0 (or the entry
  // point) changed; `untracked` = an in-place update ran (updatePoint rewrites whole neighbourhoods)
  std::vector<uint32_t> dirty0;
  bool upper_dirty = false, untracked = false;
  const float *T = nullptr;  // ADC table of the point being inserted (n_sub x Ks)

  explicit Worker(SharedBuild &s) : S(s), g(*s.g) {}

  // PQLookup (space_pq.h:16-37): sequential fp32 sum; independent of the "first" vector
  inline float dist_to_new(uint32_t id) const {
    const uint8_t *c = g.code(id);
    float r = 0.f;
    if (S.code_bytes == 1) {
      for (int m = 0; m < S.n_sub; m++) r += T[(size_t)m * S.Ks + c[m]];
    } else {
      for (int m = 0; m < S.n_sub; m++) {
        uint16_t v;
        memcpy(&v, c + 2 * m, 2);
        r += T[(size_t)m * S.Ks + v];
      }
    }
    return r;
  }

  void next_tag() {
    if (seen.size() < (size_t)g.max_elements) seen.assign((size_t)g.max_elements, 0), tag = 0;
    if (++tag == 0) {
      std::fill(seen.begin(), seen.end(), 0);
      tag = 1;
    }
  }

  // searchBaseLayer(ep, point, layer): hnswalg.h:158-238
  void search_layer(uint32_t ep, int layer, FarHeap &top) {
    next_tag();
    FarHeap &cand = h_cand;
    top.clear();
    cand.clear();
    const size_t efc = (size_t)g.ef_construction;
    float lower;
    if (!g.deleted(ep)) {
      float d = dist_to_new(ep);
      top.emplace(d, ep);
      lower = d;
      cand.emplace(-d, ep);
    } else {
      lower = std::numeric_limits<float>::max();
      cand.emplace(-lower, ep);
    }
    seen[ep] = tag;
    while (!cand.empty()) {
      Near cur = cand.top();
      if ((-cur.first) > lower) break;
      cand.pop();
      const uint32_t node = cur.second;
      // The reference holds the node's lock for the whole scan (:188).  With ~100 inserting threads every
      // walk starts at the same few hub nodes, so the lock is only held to snapshot the (<= maxM0) links and
      // the distances are evaluated outside it; single-threaded builds are unaffected (no locks at all).
      uint32_t snap[kMaxLinks];
      unsigned size;
      {
        SpinGuard lk(S.node_locks, node, S.threaded);
        uint8_t *ll = g.list_at(node, layer);
        size = std::min<unsigned>(list_count(ll), kMaxLinks);
        memcpy(snap, list_links(ll), size * sizeof(uint32_t));
      }
      const uint32_t *nb = snap;
      // every neighbour costs two cache misses (its visited tag, its code row): issue them all up front
      for (unsigned j = 0; j < size; j++) {
        __builtin_prefetch(&seen[nb[j]]);
        __builtin_prefetch(g.code(nb[j]));
      }
      for (unsigned j = 0; j < size; j++) {
        const uint32_t cid = nb[j];
        if (seen[cid] == tag) continue;
        seen[cid] = tag;
        const float d1 = dist_to_new(cid);
        if (top.size() < efc || lower > d1) {
          cand.emplace(-d1, cid);
          if (!g.deleted(cid)) top.emplace(d1, cid);
          if (top.size() > efc) top.pop();
          if (!top.empty()) lower = top.top().first;
        }
      }
      if (!cand.empty()) {  // the node expanded next (unless the loop ends): start pulling its link list
        const uint8_t *nl = g.list_at(cand.top().second, layer);
        __builtin_prefetch(nl);
        __builtin_prefetch(nl + 64);
      }
    }
  }

  // getNeighborsByHeuristic2(top_candidates, M): hnswalg.h:443-483.  In PQ mode the pairwise
  // distance inside the loop is dist_to_new(current) (SURVEY.md section 0.2).
  void select_neighbors(FarHeap &top, size_t Mlim) {
    if (top.size() < Mlim) return;
    auto &closest = h_closest;  // default less<pair>: (-(dist), id) lexicographic
    closest.clear();
    kept.clear();
    while (!top.empty()) {
      closest.emplace(-top.top().first, top.top().second);
      top.pop();
    }
    while (!closest.empty()) {
      if (kept.size() >= Mlim) break;
      Near cur = closest.top();
      const float dist_to_query = -cur.first;
      closest.pop();
      // the reference loops over `kept`, but in PQ mode its pairwise distance does not depend on the
      // kept element: it is dist_to_new(cur) every time, so one evaluation decides
      bool good = true;
      if (!kept.empty() && dist_to_new(cur.second) < dist_to_query) good = false;
      if (good) kept.push_back(cur);
    }
    for (const Near &p : kept) top.emplace(-p.first, p.second);
  }

  // mutuallyConnectNewElement(point, cur, top_candidates, level, isUpdate=false): hnswalg.h:502-619
  int connect(uint32_t cur, FarHeap &top, int level, uint32_t *next_ep, bool is_update = false) {
    const size_t Mcurmax = level ? (size_t)g.maxM : (size_t)g.maxM0;
    select_neighbors(top, (size_t)g.M);
    if (top.size() > (size_t)g.M) ANNB_FAIL(ANNB_EINVAL, "Should be not be more than M_ candidates returned by the heuristic");
    sel.clear();
    while (!top.empty()) {
      sel.push_back(top.top().second);
      top.pop();
    }
    *next_ep = sel.back();
    if (level == 0) {
      dirty0.push_back(cur);
      dirty0.insert(dirty0.end(), sel.begin(), sel.end());
    } else {
      upper_dirty = true;
    }
    {
      uint8_t *ll = g.list_at(cur, level);
      if (list_count(ll) && !is_update) ANNB_FAIL(ANNB_EINVAL, "The newly inserted element should have blank link list");
      set_list_count(ll, (unsigned)sel.size());
      uint32_t *data = list_links(ll);
      for (size_t i = 0; i < sel.size(); i++) {
        if (data[i] && !is_update) ANNB_FAIL(ANNB_EINVAL, "Possible memory corruption");
        if (level > g.levels[sel[i]]) ANNB_FAIL(ANNB_EINVAL, "Trying to make a link on a non-existent level");
        data[i] = sel[i];
      }
    }
    for (size_t i = 0; i < sel.size(); i++) {
      const uint32_t other = sel[i];
      SpinGuard lk(S.node_locks, other, S.threaded);
      uint8_t *ll = g.list_at(other, level);
      const size_t sz = list_count(ll);
      if (sz > Mcurmax) ANNB_FAIL(ANNB_EINVAL, "Bad value of sz_link_list_other");
      if (other == cur) ANNB_FAIL(ANNB_EINVAL, "Trying to connect an element to itself");
      if (level > g.levels[other]) ANNB_FAIL(ANNB_EINVAL, "Trying to make a link on a non-existent level");
      uint32_t *data = list_links(ll);
      if (is_update) {  // already linked back: leave the neighbour's list alone (:563-574)
        bool present = false;
        for (size_t j = 0; j < sz; j++)
          if (data[j] == cur) {
            present = true;
            break;
          }
        if (present) continue;
      }
      if (sz < Mcurmax) {
        data[sz] = cur;
        set_list_count(ll, (unsigned)sz + 1);
      } else {
        // "finding the weakest element": in PQ mode every distance below is dist_to_new(other)
        for (size_t j = 0; j < sz; j++) __builtin_prefetch(g.code(data[j]));  // select_neighbors scores them all
        const float d_max = dist_to_new(other);
        FarHeap &cands = h_cands;
        cands.clear();
        cands.emplace(d_max, cur);
        for (size_t j = 0; j < sz; j++) cands.emplace(dist_to_new(other), data[j]);
        select_neighbors(cands, Mcurmax);
        unsigned indx = 0;
        while (!cands.empty()) {
          data[indx++] = cands.top().second;
          cands.pop();
        }
        set_list_count(ll, indx);
      }
    }
    return ANNB_OK;
  }

  std::vector<uint32_t> connections(uint32_t id, int level) {  // getConnectionsWithLock: hnswalg.h:1098-1106
    SpinGuard lk(S.node_locks, id, S.threaded);
    uint8_t *ll = g.list_at(id, level);
    const unsigned n = list_count(ll);
    const uint32_t *d = list_links(ll);
    return std::vector<uint32_t>(d, d + n);
  }

  // repairConnectionsForUpdate: hnswalg.h:1036-1096
  int repair(uint32_t ep, uint32_t id, int elem_level, int max_level) {
    uint32_t cur_obj = ep;
    if (elem_level < max_level) {
      float curdist = dist_to_new(cur_obj);
      for (int level = max_level; level > elem_level; level--) {
        bool changed = true;
        while (changed) {
          changed = false;
          uint32_t snap[kMaxLinks];
          unsigned size;
          {
            SpinGuard lk(S.node_locks, cur_obj, S.threaded);
            uint8_t *ll = g.list_at(cur_obj, level);
            size = std::min<unsigned>(list_count(ll), kMaxLinks);
            memcpy(snap, list_links(ll), size * sizeof(uint32_t));
          }
          const uint32_t *nb = snap;
          for (unsigned i = 0; i < size; i++) {
            const uint32_t c = nb[i];
            const float d = dist_to_new(c);
            if (d < curdist) {
              curdist = d;
              cur_obj = c;
              changed = true;
            }
          }
        }
      }
    }
    if (elem_level > max_level) ANNB_FAIL(ANNB_EINVAL, "Level of item to be updated cannot be bigger than max level");
    for (int level = elem_level; level >= 0; level--) {
      FarHeap &top = h_top;
      search_layer(cur_obj, level, top);
      FarHeap &filtered = h_filtered;
      filtered.clear();
      while (!top.empty()) {
        if (top.top().second != id) filtered.push(top.top());
        top.pop();
      }
      if (!filtered.empty()) {
        if (g.deleted(ep)) {
          filtered.emplace(dist_to_new(ep), ep);
          if (filtered.size() > (size_t)g.ef_construction) filtered.pop();
        }
        int rc = connect(id, filtered, level, &cur_obj, true);
        if (rc) return rc;
      }
    }
    return ANNB_OK;
  }

  // updatePoint(point, internalId, updateNeighborProbability = 1.0): hnswalg.h:958-1034.  Re-adding an
  // existing label (AnnLite.update -> add_with_ids, annlite/container.py:343-347) lands here.  With
  // probability 1.0 the reference's update_probability_generator_ draws never skip a neighbour, so the
  // generator is not modelled.  std::unordered_set reproduces the reference's iteration order.
  int update(const uint8_t *code, uint32_t id) {
    memcpy(g.rec0(id) + g.offset_data, code, g.code_row_bytes);
    const int max_level_copy = g.maxlevel;
    const uint32_t ep_copy = g.enterpoint;
    if (ep_copy == id && g.count.load() == 1) return ANNB_OK;
    const int elem_level = g.levels[id];
    for (int layer = 0; layer <= elem_level; layer++) {
      std::unordered_set<uint32_t> s_cand, s_neigh;
      std::vector<uint32_t> one_hop = connections(id, layer);
      if (one_hop.empty()) continue;
      s_cand.insert(id);
      for (uint32_t h1 : one_hop) {
        s_cand.insert(h1);
        s_neigh.insert(h1);
        for (uint32_t h2 : connections(h1, layer)) s_cand.insert(h2);
      }
      for (uint32_t neigh : s_neigh) {
        FarHeap &cands = h_cands;
        cands.clear();
        const size_t size = s_cand.find(neigh) == s_cand.end() ? s_cand.size() : s_cand.size() - 1;
        const size_t keep = std::min((size_t)g.ef_construction, size);
        for (uint32_t c : s_cand) {
          if (c == neigh) continue;
          const float d = dist_to_new(c);  // PQLookup ignores its first argument (SURVEY.md section 0.2)
          if (cands.size() < keep) {
            cands.emplace(d, c);
          } else if (d < cands.top().first) {
            cands.pop();
            cands.emplace(d, c);
          }
        }
        select_neighbors(cands, layer == 0 ? (size_t)g.maxM0 : (size_t)g.maxM);
        SpinGuard lk(S.node_locks, neigh, S.threaded);
        uint8_t *ll = g.list_at(neigh, layer);
        const size_t n = cands.size();
        set_list_count(ll, (unsigned)n);
        uint32_t *data = list_links(ll);
        for (size_t i = 0; i < n; i++) {
          data[i] = cands.top().second;
          cands.pop();
        }
      }
    }
    return repair(ep_copy, id, elem_level, max_level_copy);
  }

  int random_level() {  // getRandomLevel: hnswalg.h:151-155
    std::uniform_real_distribution<double> distribution(0.0, 1.0);
    double r;
    if (S.threaded) {
      std::lock_guard<std::mutex> lk(S.rng_guard);
      r = -std::log(distribution(*S.level_gen)) * g.mult;
    } else {
      r = -std::log(distribution(*S.level_gen)) * g.mult;
    }
    return (int)r;
  }

  // addPoint(point, label, level=-1): hnswalg.h:1108-1235
  int insert(const float *table, const uint8_t *code, uint64_t label, int forced_level = -1) {
    T = table;
    uint32_t cur;
    {
      std::unique_lock<std::mutex> lk(S.count_guard, std::defer_lock);
      if (S.threaded) lk.lock();
      auto found = g.label_lookup.find(label);
      if (found != g.label_lookup.end()) {  // existing label: update in place (:1119-1131)
        const uint32_t existing = found->second;
        if (S.threaded) lk.unlock();
        if (g.deleted(existing)) {
          g.rec0(existing)[2] &= (uint8_t)~1;
          g.num_deleted--;
        }
        untracked = true;
        return update(code, existing);
      }
      if (g.count.load() >= g.max_elements) ANNB_FAIL(ANNB_ECAPACITY, "The number of elements exceeds the specified limit");
      cur = (uint32_t)g.count.load();
      g.count.store(cur + 1);
      g.label_lookup[label] = cur;
    }
    // held for the whole insertion like link_list_locks_[cur_c] in the reference (:1144): until every level of
    // `cur` is linked, no other thread may append itself to one of its still-blank lists
    SpinGuard self(S.node_locks, cur, S.threaded);
    const int curlevel = forced_level >= 0 ? forced_level : random_level();
    g.levels[cur] = curlevel;

    std::unique_lock<std::mutex> glk(S.global, std::defer_lock);
    if (S.threaded) glk.lock();
    const int maxlevelcopy = g.maxlevel;
    // (the reference reads enterpoint_node_ AFTER dropping the lock, hnswalg.h:1147-1151: a benign-looking race with a
    // thread that is installing a new top level; here level and entry point are read as one consistent pair)
    uint32_t cur_obj = g.enterpoint;
    const uint32_t ep_copy = cur_obj;
    if (curlevel <= maxlevelcopy && S.threaded) glk.unlock();

    uint8_t *rec = g.rec0(cur);
    memset(rec, 0, g.size_per_elem);
    memcpy(rec + g.label_offset, &label, 8);
    memcpy(rec + g.offset_data, code, g.code_row_bytes);
    if (curlevel) {
      g.upper[cur] = (uint8_t *)malloc(g.size_links_per_elem * curlevel + 1);
      if (!g.upper[cur]) ANNB_FAIL(ANNB_ENOMEM, "Not enough memory: addPoint failed to allocate linklist");
      memset(g.upper[cur], 0, g.size_links_per_elem * curlevel + 1);
    }

    if ((int32_t)cur_obj != -1) {
      if (curlevel < maxlevelcopy) {
        float curdist = dist_to_new(cur_obj);
        for (int level = maxlevelcopy; level > curlevel; level--) {
          bool changed = true;
          while (changed) {
            changed = false;
            uint32_t snap[kMaxLinks];
            unsigned size;
            {
              SpinGuard lk(S.node_locks, cur_obj, S.threaded);
              uint8_t *ll = g.list_at(cur_obj, level);
              size = std::min<unsigned>(list_count(ll), kMaxLinks);
              memcpy(snap, list_links(ll), size * sizeof(uint32_t));
            }
            const uint32_t *nb = snap;
            for (unsigned i = 0; i < size; i++) {
              const uint32_t c = nb[i];
              const float d = dist_to_new(c);
              if (d < curdist) {
                curdist = d;
                cur_obj = c;
                changed = true;
              }
            }
          }
        }
      }
      const bool ep_deleted = g.deleted(ep_copy);
      for (int level = std::min(curlevel, maxlevelcopy); level >= 0; level--) {
        FarHeap &top = h_top;
        search_layer(cur_obj, level, top);
        if (ep_deleted) {
          top.emplace(dist_to_new(ep_copy), ep_copy);
          if (top.size() > (size_t)g.ef_construction) top.pop();
        }
        int rc = connect(cur, top, level, &cur_obj);
        if (rc) return rc;
      }
    } else {
      g.enterpoint = 0;
      g.maxlevel = curlevel;
    }
    if (curlevel > maxlevelcopy) {
      g.enterpoint = cur;
      g.maxlevel = curlevel;
    }
    dirty0.push_back(cur);
    if (curlevel > 0 || (int32_t)ep_copy == -1) upper_dirty = true;
    return ANNB_OK;
  }
};

}  // namespace

// Default insertion thread count (num_threads <= 0; the reference takes hardware_concurrency(),
// hnsw_bindings.cpp:239-240).  The CPUs this process may actually run on are the smaller of the
// affinity mask and the cgroup CPU quota -- a container that reports 128 logical CPUs but is
// throttled to a fraction of them turns every held node lock into a convoy.  Capped at 32: more
// threads than that made the 1M-point build slower, not faster, on 128-thread hosts (lock convoys);
// callers that know better pass num_threads.
int hnsw_default_threads() {
  int n = (int)std::thread::hardware_concurrency();
  if (n < 1) n = 1;
#if defined(__linux__)
  cpu_set_t set;
  CPU_ZERO(&set);
  if (sched_getaffinity(0, sizeof(set), &set) == 0) {
    const int a = CPU_COUNT(&set);
    if (a > 0 && a < n) n = a;
  }
  long long quota = -1, period = -1;
  if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {  // cgroup v2: "<quota|max> <period>"
    char q[32] = {0};
    if (fscanf(f, "%31s %lld", q, &period) == 2 && strcmp(q, "max") != 0) quota = atoll(q);
    fclose(f);
  } else {
    if (FILE *fq = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
      if (fscanf(fq, "%lld", &quota) != 1) quota = -1;
      fclose(fq);
    }
    if (FILE *fp = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
      if (fscanf(fp, "%lld", &period) != 1) period = -1;
      fclose(fp);
    }
  }
  if (quota > 0 && period > 0) {
    const int c = (int)((quota + period - 1) / period);
    if (c >= 1 && c < n) n = c;
  }
#endif
  return n < 32 ? n : 32;
}

// Inserts rows [0, n) whose ADC tables are produced chunk-wise by `table_chunk(first, count)`
// (host pointer to count*M*Ks floats valid until the next call) -- see capi.cu.
int hnsw_draw_levels(annb_index *h, int64_t n, int32_t *out) {
  HostGraph &g = h->g;
  if (!g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised");
  std::uniform_real_distribution<double> distribution(0.0, 1.0);
  for (int64_t i = 0; i < n; i++) out[i] = (int32_t)(-std::log(distribution(g.level_gen)) * g.mult);
  return ANNB_OK;
}

int hnsw_insert_rows(annb_index *h, const uint8_t *codes, const uint64_t *labels, int64_t n, int num_threads,
                     const float *(*table_chunk)(void *, int64_t, int64_t), void *ctx, int64_t chunk_rows,
                     const int32_t *forced_levels, BuildTrack *track) {
  HostGraph &g = h->g;
  if (!g.inited) ANNB_FAIL(ANNB_ESTATE, "index not initialised: call annb_init_graph / annb_load_index first");
  int64_t fresh = 0;
  {
    std::unordered_set<uint64_t> seen_in_batch;
    for (int64_t i = 0; i < n; i++)
      if (g.label_lookup.find(labels[i]) == g.label_lookup.end() && seen_in_batch.insert(labels[i]).second) fresh++;
  }
  if (g.count.load() + fresh > g.max_elements) ANNB_FAIL(ANNB_ECAPACITY, "The number of elements exceeds the specified limit");
  if (num_threads <= 0) num_threads = hnsw_default_threads();
  if (fresh != n) num_threads = 1;  // updates of stored points rewrite neighbourhoods: keep them sequential
  if (num_threads < 1) num_threads = 1;
  // "avoid using threads when the number of searches is small": hnsw_bindings.cpp:242-245
  if (n <= (int64_t)num_threads * 4) num_threads = 1;

  SharedBuild S;
  S.g = &g;
  S.n_sub = h->M;
  S.Ks = h->Ks;
  S.code_bytes = h->code_bytes;
  S.threaded = num_threads > 1;
  S.level_gen = &g.level_gen;  // part of the index state: continues across add_items calls
  if (S.threaded) S.node_locks.reset((size_t)g.max_elements);
  const size_t TS = (size_t)h->M * h->Ks;
  const size_t crow = g.code_row_bytes;

  std::vector<std::unique_ptr<Worker>> workers;
  for (int t = 0; t < num_threads; t++) workers.emplace_back(new Worker(S));

  std::atomic<int> err{0};
  std::string err_msg;
  std::mutex err_mu;
  for (int64_t first = 0; first < n; first += chunk_rows) {
    const int64_t cnt = std::min(chunk_rows, n - first);
    const float *tables = table_chunk(ctx, first, cnt);
    if (!tables) return ANNB_ECUDA;
    int64_t start = 0;
    if (g.count.load() == 0 && first == 0) {  // first point alone (hnsw_bindings.cpp:266-272)
      int rc = workers[0]->insert(tables, codes, labels[0], forced_levels ? forced_levels[0] : -1);
      if (rc) return rc;
      start = 1;
    }
    if (num_threads == 1) {
      for (int64_t r = start; r < cnt; r++) {
        int rc = workers[0]->insert(tables + (size_t)r * TS, codes + (size_t)(first + r) * crow, labels[first + r],
                                    forced_levels ? forced_levels[first + r] : -1);
        if (rc) return rc;
      }
    } else {
      std::atomic<int64_t> next{start};
      std::vector<std::thread> pool;
      for (int t = 0; t < num_threads; t++) {
        pool.emplace_back([&, t] {
          Worker &w = *workers[t];
          for (;;) {
            const int64_t r = next.fetch_add(1);
            if (r >= cnt || err.load()) break;
            int rc = w.insert(tables + (size_t)r * TS, codes + (size_t)(first + r) * crow, labels[first + r],
                              forced_levels ? forced_levels[first + r] : -1);
            if (rc) {
              std::lock_guard<std::mutex> lk(err_mu);
              if (!err.load()) {
                err.store(rc);
                err_msg = annb_last_error();
              }
              break;
            }
          }
        });
      }
      for (auto &th : pool) th.join();
      if (err.load()) {
        annb_set_error("%s", err_msg.c_str());
        return err.load();
      }
    }
  }
  if (track) {
    for (auto &w : workers) {
      track->dirty0.insert(track->dirty0.end(), w->dirty0.begin(), w->dirty0.end());
      track->upper_dirty |= w->upper_dirty;
      track->untracked |= w->untracked;
    }
  }
  return ANNB_OK;
}
