#include "skch_tail.hpp"
#include <thread>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include <algorithm>
#include <atomic>
#include <charconv>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <cmath>
#include <limits>
#include <numeric>
#include <tuple>

#include "skch_filter.hpp"
#include "skch_stats.hpp"

namespace skch {

size_t MappingResult::hash() const
{  // base_types.hpp:146-151, :188-204
  size_t res = 0;
  auto combine = [&res](auto v) {
    std::hash<decltype(v)> h;
    res ^= h(v) + 0x9e3779b9 + (res << 6) + (res >> 2);
  };
  combine(queryLen); combine(refStartPos); combine(refEndPos); combine(queryStartPos); combine(queryEndPos);
  combine(refSeqId); combine(querySeqId); combine(blockLength); combine(nucIdentity); combine(nucIdentityUpperBound);
  combine(sketchSize); combine(conservedSketches); combine(strand); combine(approxMatches);
  return res;
}

IdentityCache::Table &IdentityCache::table(int qs)
{
  if (qs == last_qs) return *last;
  Table &t = tables[qs];
  if (t.identity.empty()) {
    t.identity.assign((size_t)qs + 1, std::make_pair(-1.0f, 0.0f));
    t.cutoff.assign((size_t)qs + 1, -1.0);
  }
  last = &t;  // references into an unordered_map stay valid when it grows
  last_qs = qs;
  return t;
}

std::pair<float, float> IdentityCache::get(int shared, int qs)
{
  Table &t = table(qs);
  const bool in_table = shared >= 0 && shared <= qs;
  if (in_table && t.identity[(size_t)shared].first >= 0) return t.identity[(size_t)shared];
  float mash_dist = Stat::j2md(1.0 * shared / qs, k);
  float nucIdentity = (1 - mash_dist);
  float nucIdentityUpperBound = 1 - Stat::md_lower_bound(mash_dist, qs, k, fixed::confidence_interval);
  auto v = std::make_pair(nucIdentity, nucIdentityUpperBound);
  if (in_table && nucIdentity >= 0) t.identity[(size_t)shared] = v;
  return v;
}

/* computeMap.hpp:1195-1200 for an integer-valued bestJaccardNumerator (it only ever holds 0 or a sharedSketchSize) */
double IdentityCache::cutoffJaccard(int best, int qs)
{
  Table &t = table(qs);
  const bool in_table = best >= 0 && best <= qs;
  if (in_table && t.cutoff[(size_t)best] >= 0) return t.cutoff[(size_t)best];
  const double bestJaccardNumerator = best;
  double cutoff_ani = std::max(0.0, double((1 - Stat::j2md(bestJaccardNumerator / qs, k)) - ANIDiff));
  double cutoff_j = Stat::md2j(1 - cutoff_ani, k);
  if (in_table && cutoff_j >= 0) t.cutoff[(size_t)best] = cutoff_j;
  return cutoff_j;
}

namespace {

/* union-find with the merge rule of dsets::DisjointSets (reference src/common/dset64.hpp:62-124):
 * the root of lower rank goes under the other; on equal rank the larger id goes under the smaller. */
struct UnionFind {
  std::vector<uint32_t> &parent, &rnk;  // the caller's scratch (kept between reads)
  UnionFind(size_t n, std::vector<uint32_t> &p, std::vector<uint32_t> &r) : parent(p), rnk(r)
  {
    parent.resize(n);
    rnk.assign(n, 0);
    std::iota(parent.begin(), parent.end(), 0u);
  }
  uint32_t find(uint32_t x)
  {
    while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; }
    return x;
  }
  void unite(uint32_t a, uint32_t b)
  {
    a = find(a); b = find(b);
    if (a == b) return;
    uint32_t ra = rnk[a], rb = rnk[b];
    if (ra > rb || (ra == rb && a < b)) { std::swap(ra, rb); std::swap(a, b); }
    parent[a] = b;
    if (ra == rb) rnk[b] = rb + 1;
  }
};


}  // namespace

/* ---- doL2Mapping on the device's records (computeMap.hpp:1181-1267) ---- */
void MapTail::fragmentMappings(const mm_segment &sg, const mm_segment_result &sr, const ReadRec &rd, IdentityCache &idc,
                      std::vector<mm_l1_candidate> &work, MappingResultsVector_t &l2Mappings) const
{
  l2Mappings.clear();
  if (sr.sketch_raw_count == 0 || sr.sketch_size == 0) return;  // :822-825, :1136
  // Q.kmerComplexity (computeMap.hpp:830-831): long double ratio -> double -> float
  const double max_hash_01 = (long double)(sr.sketch_max_hash) / std::numeric_limits<hash_t>::max();
  const float kmerComplexity = (double(sr.sketch_raw_count) / max_hash_01) / ((sg.length - param.kmerSize + 1) * 2);
  if (kmerComplexity < param.kmerComplexityThreshold) return;  // :1136
  if (sr.n_candidates == 0) return;
  const int qs = sr.sketch_size;
  work.assign(cands + sr.first_candidate, cands + sr.first_candidate + sr.n_candidates);
  auto cmp = [](const mm_l1_candidate &a, const mm_l1_candidate &b) { return a.intersectionSize < b.intersectionSize; };
  size_t gb = 0;
  while (gb < work.size()) {  // mapSingleQueryFrag's per-reference-group loop (:772-797)
    size_t ge = work.size();
    if (param.skip_prefix) {
      const int g = refIdGroup[work[gb].seqId];
      ge = gb;
      while (ge < work.size() && refIdGroup[work[ge].seqId] == g) ge++;
    }
    if (param.stage1_topANI_filter) std::make_heap(work.begin() + gb, work.begin() + ge, cmp);
    double bestJaccardNumerator = 0;
    size_t it = gb, end = ge;
    while (it != end) {
      const mm_l1_candidate &cd = work[it];
      if (param.stage1_topANI_filter) {
        const double cutoff_j = idc.cutoffJaccard((int)bestJaccardNumerator, qs);
        if (double(cd.intersectionSize) / qs < cutoff_j) break;
      }
      for (uint32_t li = 0; li < cd.n_loci; li++) {
        const mm_l2_locus &l2 = loci[cd.first_locus + li];
        const auto id = idc.get(l2.sharedSketchSize, qs);
        const float nucIdentity = id.first, nucIdentityUpperBound = id.second;
        if ((param.keep_low_pct_id && nucIdentityUpperBound >= param.percentageIdentity) ||
            nucIdentity >= param.percentageIdentity) {
          bestJaccardNumerator = std::max<double>(bestJaccardNumerator, l2.sharedSketchSize);
          MappingResult res{};
          res.n_merged = 1;  // see skch_tail.hpp: the reference leaves this uninitialised
          res.queryLen = sg.length;
          res.refStartPos = l2.meanOptimalPos;
          res.refEndPos = l2.meanOptimalPos + sg.length;
          res.queryStartPos = 0;
          res.queryEndPos = sg.length;
          res.refSeqId = l2.seqId;
          res.querySeqId = rd.seqCounter;
          res.nucIdentity = nucIdentity;
          res.nucIdentityUpperBound = nucIdentityUpperBound;
          res.sketchSize = qs;
          res.conservedSketches = l2.sharedSketchSize;
          res.blockLength = std::max(res.refEndPos - res.refStartPos, res.queryEndPos - res.queryStartPos);
          res.approxMatches = std::round(res.nucIdentity * res.blockLength / 100.0);
          res.strand = (strand_t)l2.strand;
          res.kmerComplexity = kmerComplexity;
          res.selfMapFilter = ((param.skip_self || param.skip_prefix) && rd.len > metadata[l2.seqId].len);
          l2Mappings.push_back(res);
        }
      }
      if (param.stage1_topANI_filter) {
        std::pop_heap(work.begin() + gb, work.begin() + end, cmp);
        end--;
      } else {
        it++;
      }
    }
    gb = ge;
  }
  std::sort(l2Mappings.begin(), l2Mappings.end(), [](const MappingResult &a, const MappingResult &b) {
    return std::tie(a.refSeqId, a.refStartPos) < std::tie(b.refSeqId, b.refStartPos);
  });  // :800-801
}

/* ---- mergeMappingsInRange (computeMap.hpp:1579-1704) ---- */
void MapTail::mergeMappingsInRange(MappingResultsVector_t &readMappings, int max_dist) const
{
  if (readMappings.size() < 2) return;
  std::sort(readMappings.begin(), readMappings.end(), [](const MappingResult &a, const MappingResult &b) {
    return std::tie(a.refSeqId, a.refStartPos, a.queryStartPos) < std::tie(b.refSeqId, b.refStartPos, b.queryStartPos);
  });
  for (size_t i = 0; i < readMappings.size(); i++) { readMappings[i].splitMappingId = (offset_t)i; readMappings[i].discard = 0; }
  static thread_local std::vector<uint32_t> uf_parent, uf_rank;  // per-worker scratch: no allocation per read once warm
  static thread_local std::vector<std::pair<double, uint64_t>> distances;
  UnionFind uf(readMappings.size(), uf_parent, uf_rank);
  for (auto it = readMappings.begin(); it != readMappings.end(); it++) {
    distances.clear();
    for (auto it2 = std::next(it); it2 != readMappings.end(); it2++) {
      if (it2->refSeqId != it->refSeqId || it2->refStartPos > it->refEndPos + max_dist) break;
      if (it2->strand == it->strand) {
        int ref_dist = it2->refStartPos - it->refEndPos;
        int query_dist = 0;
        auto dist = std::numeric_limits<double>::max();
        auto score = std::numeric_limits<double>::max();
        if (it->strand == strnd::FWD && it->queryStartPos <= it2->queryStartPos) {
          query_dist = it2->queryStartPos - it->queryEndPos;
          dist = std::sqrt(std::pow(query_dist, 2) + std::pow(ref_dist, 2));
          score = std::pow(query_dist - ref_dist, 2);
        } else if (it->strand != strnd::FWD && it->queryEndPos >= it2->queryEndPos) {
          query_dist = it->queryStartPos - it2->queryEndPos;
          dist = std::sqrt(std::pow(query_dist, 2) + std::pow(ref_dist, 2));
          score = std::pow(query_dist - ref_dist, 2);
        }
        if (dist < max_dist) distances.push_back(std::make_pair(dist + score, (uint64_t)it2->splitMappingId));
      }
    }
    if (distances.size()) {
      std::sort(distances.begin(), distances.end());
      uf.unite((uint32_t)it->splitMappingId, (uint32_t)distances.front().second);
    }
  }
  for (auto &m : readMappings) m.splitMappingId = (offset_t)uf.find((uint32_t)m.splitMappingId);
  std::sort(readMappings.begin(), readMappings.end(),
            [](const MappingResult &a, const MappingResult &b) { return a.splitMappingId < b.splitMappingId; });
  for (auto it = readMappings.begin(); it != readMappings.end();) {
    auto it_end = std::find_if(it, readMappings.end(), [&](const MappingResult &e) { return e.splitMappingId != it->splitMappingId; });
    std::for_each(it, it_end, [&](MappingResult &e) {
      it->queryStartPos = std::min(it->queryStartPos, e.queryStartPos);
      it->refStartPos = std::min(it->refStartPos, e.refStartPos);
      it->queryEndPos = std::max(it->queryEndPos, e.queryEndPos);
      it->refEndPos = std::max(it->refEndPos, e.refEndPos);
      it->blockLength = std::max(it->refEndPos - it->refStartPos, it->queryEndPos - it->queryStartPos);
      it->approxMatches = std::round(it->nucIdentity * it->blockLength / 100.0);
    });
    it->n_merged = std::distance(it, it_end);
    it->nucIdentity = (std::accumulate(it, it_end, 0.0, [](double x, MappingResult &e) { return x + e.nucIdentity; })) / it->n_merged;
    it->kmerComplexity = (std::accumulate(it, it_end, 0.0, [](double x, MappingResult &e) { return x + e.kmerComplexity; })) / it->n_merged;
    std::for_each(std::next(it), it_end, [&](MappingResult &e) { e.discard = 1; });
    it = it_end;
  }
  readMappings.erase(std::remove_if(readMappings.begin(), readMappings.end(), [](MappingResult &e) { return e.discard == 1; }),
                     readMappings.end());
}

/* ---- std::sort's permutation, computed faster ----
 * The run-wide one-to-one step sorts ALL mappings four times with std::sort, and what it writes depends on how std::sort
 * leaves records with EQUAL keys (the reference-axis sweep refuses a mapping equivalent to one already in its status, and
 * which of two equivalent mappings comes first is decided by these sorts). So the product must end up with exactly the
 * arrangement libstdc++'s introsort gives the reference. Three things make that cheap without changing it:
 *  (1) the sort runs on (key, index) pairs and the 96-byte records are permuted once afterwards -- introsort decides every
 *      move from comparison results alone, so the pairs end up arranged as the records would;
 *  (2) the key tuple is packed into unsigned words whose order is the tuple's lexicographic order (int32 fields biased by
 *      2^31): same comparison results, fewer instructions and no branches per comparison;
 *  (3) the quicksort phase runs on several threads. __introsort_loop partitions a range and then treats the two sides
 *      independently; everything left of a cut is <= everything right of it, so the final insertion pass never moves a
 *      record across a cut either. Handing the right-hand side of a cut to another thread therefore changes nothing but
 *      the order in which disjoint ranges are processed. The code below calls libstdc++'s own partition / loop / heap /
 *      insertion routines (bits/stl_algo.h), it does not restate them; other standard libraries take the serial std::sort. */
namespace {

inline uint32_t biased(int32_t x) { return (uint32_t)x ^ 0x80000000u; }
inline uint64_t pack2(int32_t a, int32_t b) { return ((uint64_t)biased(a) << 32) | biased(b); }

/* packed (alignment 1): they live inside packed (key, index) pairs at any offset */
struct Key2 {  // (a, b)
  uint64_t k;
  bool operator<(const Key2 &o) const { return k < o.k; }
} __attribute__((packed));
struct Key3 {  // (a, b, c)
  uint64_t hi;
  uint32_t lo;
  bool operator<(const Key3 &o) const { return hi < o.hi || (hi == o.hi && lo < o.lo); }
} __attribute__((packed));
struct Key4 {  // (a, b, c, d)
  uint64_t hi, lo;
  bool operator<(const Key4 &o) const { return hi < o.hi || (hi == o.hi && lo < o.lo); }
} __attribute__((packed));
inline Key2 key_ref(const MappingResult &m) { return Key2{pack2(m.refSeqId, m.refStartPos)}; }
inline Key3 key_query_ref(const MappingResult &m) { return Key3{pack2(m.queryStartPos, m.refSeqId), biased(m.refStartPos)}; }
inline Key4 key_read_query_ref(const MappingResult &m)
{
  return Key4{pack2(m.querySeqId, m.queryStartPos), pack2(m.refSeqId, m.refStartPos)};
}

/* a handful of helper threads for one call; jobs may enqueue jobs */
class JobPool {
 public:
  explicit JobPool(int threads) : threads_(threads) {}
  void add(std::function<void()> fn)
  {
    {
      std::lock_guard<std::mutex> g(m_);
      q_.push_back(std::move(fn));
      pending_++;
    }
    cv_.notify_one();
  }
  void finish()  // helpers start now (the first jobs are queued); the caller works too, until every job (and the jobs they added) is done
  {
    for (int t = 1; t < threads_; t++) pool_.emplace_back([this] { run(); });
    run();
    for (auto &th : pool_) th.join();
    pool_.clear();
  }

 private:
  void run()
  {
    std::unique_lock<std::mutex> g(m_);
    while (true) {
      if (!q_.empty()) {
        auto fn = std::move(q_.back());
        q_.pop_back();
        g.unlock();
        fn();
        g.lock();
        if (--pending_ == 0) cv_.notify_all();
      } else if (pending_ == 0) {
        return;
      } else {
        cv_.wait(g);
      }
    }
  }
  std::mutex m_;
  std::condition_variable cv_;
  std::vector<std::function<void()>> q_;
  size_t pending_ = 0;
  int threads_;
  std::vector<std::thread> pool_;
};

std::atomic<long> g_heapSortBranch{0};  // how often the threaded sort took introsort's heap-sort branch (self-test evidence)

#if defined(__GLIBCXX__)
template <class P, class Cmp>
void introsortJob(P *first, P *last, long depth, Cmp cmp, JobPool &pool, long grain)
{  // std::__introsort_loop(first, last, depth, cmp) with the recursive call given away, then the insertion pass of what is left
  while (last - first > 16) {  // _S_threshold
    if (last - first <= grain) {
      std::__introsort_loop(first, last, depth, cmp);
      break;
    }
    if (depth == 0) {
      g_heapSortBranch.fetch_add(1, std::memory_order_relaxed);
      std::__partial_sort(first, last, last, cmp);
      break;
    }
    --depth;
    P *cut = std::__unguarded_partition_pivot(first, last, cmp);
    P *rlast = last;
    pool.add([=, &pool] { introsortJob(cut, rlast, depth, cmp, pool, grain); });
    last = cut;
  }
  std::__insertion_sort(first, last, cmp);
}
#endif

/* p[0..n) arranged as std::sort(p, p + n, less) arranges it */
template <class P, class Less>
void sortExactlyLikeStd(P *p, size_t n, Less less, int threads)
{
#if defined(__GLIBCXX__)
  if (threads > 1 && n >= 32768) {
    auto cmp = __gnu_cxx::__ops::__iter_comp_iter(less);
    JobPool pool(threads);
    const long grain = (long)std::max<size_t>(4096, n / ((size_t)threads * 8));
    const long depth = std::__lg((long)n) * 2;
    pool.add([=, &pool] { introsortJob(p, p + n, depth, cmp, pool, grain); });
    pool.finish();
    return;
  }
#endif
  std::sort(p, p + n, less);
}

template <class Fn>
void inSlices(size_t n, int T, Fn fn)  // fn(lo, hi) over [0, n) on T threads
{
  std::vector<std::thread> pool;
  for (int t = 1; t < T; t++) pool.emplace_back([&, t] { fn(n * (size_t)t / (size_t)T, n * (size_t)(t + 1) / (size_t)T); });
  fn(0, n / (size_t)T);
  for (auto &th : pool) th.join();
}

}  // namespace

/* std::sort(v, key(a) < key(b)): see above. `key` returns one of the packed keys. With drop_discarded, records whose
 * `discard` flag is set are erased first (remove_if keeps the others in order, and so does leaving them out of the pairs). */
template <class KeyFn>
static void sortLikeStd(MappingResultsVector_t &v, KeyFn key, int threads = 1, bool drop_discarded = false)
{
  typedef decltype(key(v[0])) K;
  if (v.size() < 2048) {
    if (drop_discarded) v.erase(std::remove_if(v.begin(), v.end(), [](const MappingResult &e) { return e.discard == 1; }), v.end());
    std::sort(v.begin(), v.end(), [&](const MappingResult &a, const MappingResult &b) { return key(a) < key(b); });
    return;
  }
  struct P { K k; uint32_t i; } __attribute__((packed));
  size_t n = v.size();
  const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, threads), n / 16384));
  static thread_local std::vector<P> p;                    // scratch kept between calls: no 14 MB of fresh pages per sort
  static thread_local MappingResultsVector_t out;
  p.resize(n);
  P *pp = p.data();  // the helper threads must see THIS thread's scratch, not their own (empty) thread_local copies
  const MappingResult *vv = v.data();
  inSlices(n, T, [&](size_t lo, size_t hi) { for (size_t i = lo; i < hi; i++) { pp[i].k = key(vv[i]); pp[i].i = (uint32_t)i; } });
  if (drop_discarded) {
    size_t m = 0;
    for (size_t i = 0; i < n; i++)
      if (!vv[i].discard) pp[m++] = pp[i];
    n = m;
  }
  sortExactlyLikeStd(pp, n, [](const P &a, const P &b) { return a.k < b.k; }, T);
  out.resize(n);
  MappingResult *oo = out.data();
  inSlices(n, T, [&](size_t lo, size_t hi) { for (size_t i = lo; i < hi; i++) oo[i] = vv[pp[i].i]; });
  v.swap(out);
}

/* Self-test of sortExactlyLikeStd against std::sort on (key, index) pairs, n elements, `threads` threads.
 * pattern 0: random keys from a small range (many ties); 1: ascending; 2: descending; 3: organ pipe; 4: all equal;
 * 5, 6: an adversarial input built with McIlroy's "antiqsort" construction against libstdc++'s own std::sort (keys are decided
 *    while std::sort runs, so that every pivot it picks is nearly the smallest key left): quicksort degenerates, the depth
 *    limit is reached and the heap-sort branch (__partial_sort) of the threaded version runs, on ranges of every size.
 * Returns the number of positions at which the two arrangements differ; *heap_branches = how often the threaded sort took
 * the heap-sort branch. */
int64_t MapTail::sortSelftest(int64_t n64, uint64_t seed, int threads, int pattern, int64_t *heap_branches)
{
  struct P { uint64_t k; uint32_t i; } __attribute__((packed));
  const long heap0 = g_heapSortBranch.load();
  const size_t n = (size_t)n64;
  uint64_t x = seed * 0x9E3779B97F4A7C15ULL + 777;
  auto rnd = [&]() { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
  std::vector<uint64_t> key(n);
  switch (pattern) {
    case 0: for (auto &k : key) k = rnd() % 1000; break;
    case 1: for (size_t i = 0; i < n; i++) key[i] = i / 3; break;
    case 2: for (size_t i = 0; i < n; i++) key[i] = (n - i) / 3; break;
    case 3: for (size_t i = 0; i < n; i++) key[i] = std::min(i, n - 1 - i) / 2; break;
    case 4: for (auto &k : key) k = 42; break;
    default: {
      /* antiqsort: items start as "gas" (undecided, larger than every decided key); a comparison of two gas items freezes
       * the one that was a recent pivot candidate to the next solid value */
      const uint64_t gas = (uint64_t)n;
      std::vector<uint64_t> val(n, gas);
      std::vector<uint32_t> ptr(n);
      for (size_t i = 0; i < n; i++) ptr[i] = (uint32_t)i;
      uint64_t nsolid = 0;
      uint32_t candidate = 0;
      std::sort(ptr.begin(), ptr.end(), [&](uint32_t a, uint32_t b) {
        if (val[a] == gas && val[b] == gas) {
          if (a == candidate) val[a] = nsolid++;
          else val[b] = nsolid++;
        }
        if (val[a] == gas) candidate = a;
        else if (val[b] == gas) candidate = b;
        return val[a] < val[b];
      });
      for (size_t i = 0; i < n; i++) key[i] = (val[i] == gas ? nsolid : val[i]) / (pattern == 6 ? 2 : 1);  // 6: halved, ties as well
    }
  }
  std::vector<P> a(n), b(n);
  for (size_t i = 0; i < n; i++) { a[i].k = key[i]; a[i].i = (uint32_t)i; }
  b = a;
  auto less = [](const P &l, const P &r) { return l.k < r.k; };
  std::sort(a.begin(), a.end(), less);
  sortExactlyLikeStd(b.data(), n, less, threads);
  int64_t bad = 0;
  for (size_t i = 0; i < n; i++) bad += a[i].i != b[i].i;
  if (heap_branches) *heap_branches = g_heapSortBranch.load() - heap0;
  return bad;
}

/* ---- filterByGroup (computeMap.hpp:504-561) ---- */
void MapTail::filterByGroup(MappingResultsVector_t &unfiltered, MappingResultsVector_t &filtered, int n_mappings, bool filter_ref) const
{
  filtered.reserve(unfiltered.size());
  const bool trace = filter_ref && getenv("MM_TRACE") != nullptr;
  auto tt0 = std::chrono::steady_clock::now();
  auto lap = [&](const char *what) {
    if (!trace) return;
    auto t = std::chrono::steady_clock::now();
    fprintf(stderr, "[trace]   filterByGroup %s: %.1f ms\n", what, std::chrono::duration<double, std::milli>(t - tt0).count());
    tt0 = t;
  };
  const int sort_threads = filter_ref ? param.threads : 1;  // the run-wide step only: the per-read calls are far below the threshold
  sortLikeStd(unfiltered, key_ref, sort_threads);
  lap("sort 1");
  auto sb = unfiltered.begin(), se = unfiltered.begin();
  if (param.filterMode == filter::MAP || param.filterMode == filter::ONETOONE) {
    MappingResultsVector_t tmp;
    while (se != unfiltered.end()) {
      if (param.skip_prefix) {
        const int g = refIdGroup[sb->refSeqId];
        se = std::find_if_not(sb, unfiltered.end(), [&](const MappingResult &c) { return g == refIdGroup[c.refSeqId]; });
      } else {
        se = unfiltered.end();
      }
      tmp.insert(tmp.end(), std::make_move_iterator(sb), std::make_move_iterator(se));
      sortLikeStd(tmp, key_query_ref, sort_threads);
      lap("sort 2");
      if (filter_ref) Filter::ref::filterMappingsParallel(tmp, metadata, (uint16_t)n_mappings, param.threads);
      else Filter::query::filterMappings(tmp, (uint16_t)n_mappings);
      lap("sweep");
      filtered.insert(filtered.end(), std::make_move_iterator(tmp.begin()), std::make_move_iterator(tmp.end()));
      tmp.clear();
      sb = se;
    }
  }
  sortLikeStd(filtered, key_query_ref, sort_threads);
}

int MapTail::getRefGroup(const std::string &seqName) const
{  // computeMap.hpp:164-177
  const auto queryPrefix = seqName.substr(0, seqName.find_last_of(param.prefix_delim));
  for (size_t i = 0; i < metadata.size(); i++)
    if (queryPrefix == metadata[i].name.substr(0, metadata[i].name.find_last_of(param.prefix_delim))) return refIdGroup[i];
  return -1;
}

/* -f one-to-one, the run-wide step of mapQuery (computeMap.hpp:358-405) */
void MapTail::finalizeOneToOne(MappingResultsVector_t &allReadMappings, const std::vector<ContigInfo> &qmeta, std::string &paf) const
{
  const bool trace = getenv("MM_TRACE") != nullptr;
  auto tt0 = std::chrono::steady_clock::now();
  auto lap = [&](const char *what) {
    if (!trace) return;
    auto t = std::chrono::steady_clock::now();
    fprintf(stderr, "[trace] one-to-one %s: %.1f ms\n", what, std::chrono::duration<double, std::milli>(t - tt0).count());
    tt0 = t;
  };
  const int n_mappings = param.numMappingsForSegment - 1;
  if (!param.skip_prefix) {
    /* one group of queries and one of references: filterByGroup's steps (:504-561) on the vector itself -- the general
     * path below copies the ten megabytes of records of a 100 k-read run four times into freshly allocated vectors */
    const bool tr2 = trace;
    auto lap2 = [&](const char *what) { if (tr2) lap(what); };
    sortLikeStd(allReadMappings, key_ref, param.threads);
    lap2("  sort by reference position");
    sortLikeStd(allReadMappings, key_query_ref, param.threads);
    lap2("  sort by query start");
    Filter::ref::filterMappingsParallel(allReadMappings, metadata, (uint16_t)n_mappings, param.threads, false);
    lap2("  sweep");
    sortLikeStd(allReadMappings, key_query_ref, param.threads, true);  // drops what the sweep discarded
    lap2("  sort by query start again");
  } else {
    auto sb = allReadMappings.begin(), se = allReadMappings.begin();
    MappingResultsVector_t tmp, filtered;
    while (se != allReadMappings.end()) {
      const int g = getRefGroup(qmeta[sb->querySeqId].name);
      se = std::find_if_not(sb, allReadMappings.end(), [&](const MappingResult &c) { return g == getRefGroup(qmeta[c.querySeqId].name); });
      tmp.insert(tmp.end(), std::make_move_iterator(sb), std::make_move_iterator(se));
      filterByGroup(tmp, filtered, n_mappings, true);
      tmp.clear();
      sb = se;
    }
    allReadMappings = std::move(filtered);
  }
  lap("filterByGroup");
  sortLikeStd(allReadMappings, key_read_query_ref, param.threads);
  lap("final sort");
  /* the PAF text: formatted in slices by the host threads and joined in order (every slice starts from a stream in its
   * default state, as the single stream of the reference is for every line) */
  MapTail t(param, metadata, refIdGroup);
  t.qmetadata = &qmeta;
  const size_t n = allReadMappings.size();
  if (trace) fprintf(stderr, "[trace] one-to-one %zu mappings kept\n", n);
  const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, param.threads), n / 2048));
  std::vector<std::string> &part = textParts;  // kept between calls: no fresh pages for 10 MB of text every run
  if (part.size() < (size_t)T) part.resize((size_t)T);
  std::vector<size_t> at((size_t)T + 1, 0);
  auto fmt = [&](int ti) {
    const size_t lo = n * (size_t)ti / (size_t)T, hi = n * (size_t)(ti + 1) / (size_t)T;
    /* the string OBJECT a thread appends to lives on its own stack: the headers of part[0..T) sit next to each other in
     * one vector and every append writes the length field (no false sharing between the formatting threads) */
    std::string mine = std::move(part[(size_t)ti]);
    mine.clear();
    t.formatMappings(allReadMappings.data() + lo, hi - lo, "", mine);
    part[(size_t)ti] = std::move(mine);
  };
  {
    std::vector<std::thread> pool;
    for (int ti = 1; ti < T; ti++) pool.emplace_back(fmt, ti);
    fmt(0);
    for (auto &th : pool) th.join();
  }
  lap("text: format");
  for (int ti = 0; ti < T; ti++) at[(size_t)ti + 1] = at[(size_t)ti] + part[(size_t)ti].size();
  paf.resize(at[(size_t)T]);
  char *dst = &paf[0];
  auto join = [&](int ti) { memcpy(dst + at[(size_t)ti], part[(size_t)ti].data(), part[(size_t)ti].size()); };
  {
    std::vector<std::thread> pool;
    for (int ti = 1; ti < T; ti++) pool.emplace_back(join, ti);
    join(0);
    for (auto &th : pool) th.join();
  }
  lap("text");
}

/* ---- mapModule for one read, given the device results of its fragments (computeMap.hpp:570-714) ---- */
void MapTail::mapRead(const ReadRec &rd, IdentityCache &idc, MappingResultsVector_t &out) const
{
  MappingResultsVector_t &unfiltered = idc.unfiltered, &l2Mappings = idc.l2Mappings;
  std::vector<mm_l1_candidate> &work = idc.work;
  unfiltered.clear(); l2Mappings.clear(); work.clear();
  bool split_mapping = true;
  if (!param.split || rd.len <= param.segLength) {  // :587-607: one fragment of the whole read
    fragmentMappings(segs[rd.first_seg], segRes[rd.first_seg], rd, idc, work, l2Mappings);
    unfiltered.insert(unfiltered.end(), l2Mappings.begin(), l2Mappings.end());
    split_mapping = false;
  } else {
    const int noOverlapFragmentCount = rd.len / param.segLength;
    for (int i = 0; i < noOverlapFragmentCount; i++) {  // :613-641
      fragmentMappings(segs[rd.first_seg + i], segRes[rd.first_seg + i], rd, idc, work, l2Mappings);
      for (auto &e : l2Mappings) {
        e.queryLen = rd.len;
        e.queryStartPos = i * param.segLength;
        e.queryEndPos = i * param.segLength + param.segLength;
      }
      unfiltered.insert(unfiltered.end(), l2Mappings.begin(), l2Mappings.end());
    }
    if (noOverlapFragmentCount >= 1 && rd.len % param.segLength != 0) {  // :644-671
      const uint64_t s = rd.first_seg + noOverlapFragmentCount;
      fragmentMappings(segs[s], segRes[s], rd, idc, work, l2Mappings);
      for (auto &e : l2Mappings) {
        e.queryLen = rd.len;
        e.queryStartPos = rd.len - param.segLength;
        e.queryEndPos = rd.len;
      }
      unfiltered.insert(unfiltered.end(), l2Mappings.begin(), l2Mappings.end());
    }
  }
  const int n_mappings = (rd.len < param.segLength ? param.numMappingsForShortSequence : param.numMappingsForSegment) - 1;
  if (split_mapping && param.mergeMappings) {
    mergeMappingsInRange(unfiltered, param.chain_gap);
    const int64_t min_count = std::floor(param.block_length / param.segLength);  // filterWeakMappings :423-433
    unfiltered.erase(std::remove_if(unfiltered.begin(), unfiltered.end(),
                                    [&](MappingResult &e) { return e.queryLen > e.blockLength && e.n_merged < min_count; }),
                     unfiltered.end());
  }
  if (param.filterMode == filter::MAP || param.filterMode == filter::ONETOONE) {
    MappingResultsVector_t &tmp = idc.filtered;
    tmp.clear();
    filterByGroup(unfiltered, tmp, n_mappings, false);
    unfiltered.swap(tmp);
  }
  out.assign(unfiltered.begin(), unfiltered.end());  // `out` keeps the capacity it had for the previous batch's read
  if (param.filterLengthMismatches) {  // filterFalseHighIdentity :441-454
    out.erase(std::remove_if(out.begin(), out.end(),
                             [&](MappingResult &e) {
                               int64_t q_l = (int64_t)e.queryEndPos - (int64_t)e.queryStartPos;
                               int64_t r_l = (int64_t)e.refEndPos + 1 - (int64_t)e.refStartPos;
                               uint64_t delta = std::abs(r_l - q_l);
                               float len_id_bound = (1.0 - (float)delta / (float)q_l);
                               return len_id_bound < std::min(0.7, std::pow(param.percentageIdentity, 3));
                             }),
              out.end());
  }
  for (auto &e : out) {  // mappingBoundarySanityCheck :1713-1750
    const offset_t rlen = metadata[e.refSeqId].len;
    if (e.refStartPos < 0) e.refStartPos = 0;
    if (e.refStartPos >= rlen) e.refStartPos = rlen - 1;
    if (e.refEndPos < e.refStartPos) e.refEndPos = e.refStartPos;
    if (e.refEndPos >= rlen) e.refEndPos = rlen - 1;
    if (e.queryStartPos < 0) e.queryStartPos = 0;
    if (e.queryStartPos >= rd.len) e.queryStartPos = rd.len;
    if (e.queryEndPos < e.queryStartPos) e.queryEndPos = e.queryStartPos;
    if (e.queryEndPos >= rd.len) e.queryEndPos = rd.len;
  }
  if (param.sparsity_hash_threshold < std::numeric_limits<uint64_t>::max()) {  // sparsifyMappings :482-493
    out.erase(std::remove_if(out.begin(), out.end(), [&](MappingResult &e) { return e.hash() > param.sparsity_hash_threshold; }),
              out.end());
  }
}

/* ---- reportReadMappings (computeMap.hpp:1758-1805): same stream formatting ---- */
/* reportReadMappings (computeMap.hpp:1758-1805) through an ostream, as the reference writes it: kept as the plain statement
 * the fast formatter below is tested against (tests/test_host_cpu.py) */
void MapTail::formatMappingsStream(const MappingResultsVector_t &readMappings, const std::string &queryName, std::ostream &os) const
{
  for (auto &e : readMappings) {
    float fakeMapQ = e.nucIdentity == 1 ? 255 : std::round(-10.0 * std::log10(1 - (e.nucIdentity)));
    std::string sep = param.legacy_output ? " " : "\t";
    os << (param.filterMode == filter::ONETOONE ? (*qmetadata)[e.querySeqId].name : queryName) << sep << e.queryLen << sep
       << e.queryStartPos << sep << e.queryEndPos - (param.legacy_output ? 1 : 0) << sep
       << (e.strand == strnd::FWD ? "+" : "-") << sep << metadata[e.refSeqId].name << sep
       << metadata[e.refSeqId].len << sep << e.refStartPos << sep << e.refEndPos - (param.legacy_output ? 1 : 0);
    if (!param.legacy_output) {
      os << sep << e.conservedSketches << sep << e.blockLength << sep << fakeMapQ << sep << "id:f:"
         << (param.report_ANI_percentage ? 100.0 : 1.0) * e.nucIdentity << sep << "kc:f:" << e.kmerComplexity;
      if (!param.mergeMappings) os << sep << "jc:f:" << float(e.conservedSketches) / e.sketchSize;
    } else {
      os << sep << e.nucIdentity * 100.0;
    }
    os << "\n";
  }
}

namespace {
/* what `os << v` writes for an integer / a floating-point value on a default-formatted stream: decimal digits, and
 * printf's %g with precision 6 (std::to_chars(general, 6) is specified as exactly that conversion) */
inline void put_int(std::string &out, long long v)
{
  char buf[24];
  auto r = std::to_chars(buf, buf + sizeof(buf), v);
  out.append(buf, r.ptr);
}
/* printf's %g with precision 6 for 1e-3 <= v < 1e6 without the general-purpose conversion (three of these per PAF line
 * were most of the formatting time): scale to six significant digits, round to nearest-even, strip trailing zeros. The
 * scaling v * 10^(5-e) is checked to be EXACT (fma residue 0), so the rounding sees the true value -- ties of dyadic
 * identities included -- and anything else (other magnitudes, inexact products, nan, inf, zero, negatives) takes
 * std::to_chars. Returns the end of the text, or nullptr when it declines. */
inline char *g6_fast(char *buf, double v)
{
  if (!(v >= 1e-3 && v < 1e6)) return nullptr;
  static const double p10[9] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8};
  int e = v >= 1e3 ? (v >= 1e5 ? 5 : v >= 1e4 ? 4 : 3)
                   : v >= 1e0 ? (v >= 1e2 ? 2 : v >= 1e1 ? 1 : 0) : (v >= 1e-1 ? -1 : v >= 1e-2 ? -2 : -3);
  const double scale = p10[5 - e];
  const double p = v * scale;
  if (std::fma(v, scale, -p) != 0.0) return nullptr;
  long n = (long)std::nearbyint(p);  // round-half-even (default rounding mode) of an exact value
  if (n < 100000 || n > 1000000) return nullptr;  // a threshold constant on the wrong side of its power of ten
  if (n == 1000000) { n = 100000; e++; }
  if (e > 5) return nullptr;  // rounds up to 1e+06
  char d[6];
  for (int i = 5; i >= 0; i--) { d[i] = (char)('0' + n % 10); n /= 10; }
  int last = 5;
  while (last > 0 && d[last] == '0') last--;  // %g drops trailing zeros (d[0] is never 0)
  char *o = buf;
  if (e >= 0) {
    for (int i = 0; i <= e; i++) *o++ = d[i];
    if (last > e) {
      *o++ = '.';
      for (int i = e + 1; i <= last; i++) *o++ = d[i];
    }
  } else {
    *o++ = '0'; *o++ = '.';
    for (int i = 0; i < -e - 1; i++) *o++ = '0';
    for (int i = 0; i <= last; i++) *o++ = d[i];
  }
  return o;
}
template <class F>
inline void put_real(std::string &out, F v)
{
  char buf[64];
  const double dv = (double)v;
  if ((F)dv == v) {  // always for float and double; a long double kmerComplexity holds a float or a mean computed in double
    if (char *e = g6_fast(buf, dv)) { out.append(buf, e); return; }
    /* same value, same text -- and the double conversion is lock-free, while libstdc++ prints a long double through
     * snprintf under a freshly created "C" locale (newlocale / freelocale take a process-wide lock on every call: 16
     * formatting threads ran at the speed of one) */
    auto r = std::to_chars(buf, buf + sizeof(buf), dv, std::chars_format::general, 6);
    out.append(buf, r.ptr);
    return;
  }
  auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::general, 6);
  out.append(buf, r.ptr);
}
}  // namespace

/* The same text appended to a string without a stream: the PAF lines were 3/4 of the host tail's time per read
 * (scripts/tail_perf.py: 1.25 of 1.65 us), and at N GPUs on one host the tail is what the host CPUs are short of. */
void MapTail::formatMappings(const MappingResultsVector_t &readMappings, const std::string &queryName, std::string &out) const
{
  formatMappings(readMappings.data(), readMappings.size(), queryName, out);
}

void MapTail::formatMappings(const MappingResult *first, size_t n, const std::string &queryName, std::string &out) const
{
  const char sep = param.legacy_output ? ' ' : '\t';
  for (const MappingResult *it = first; it != first + n; ++it) {
    const MappingResult &e = *it;
    const float fakeMapQ = e.nucIdentity == 1 ? 255 : std::round(-10.0 * std::log10(1 - (e.nucIdentity)));
    out += (param.filterMode == filter::ONETOONE ? (*qmetadata)[e.querySeqId].name : queryName);
    out += sep; put_int(out, e.queryLen);
    out += sep; put_int(out, e.queryStartPos);
    out += sep; put_int(out, e.queryEndPos - (param.legacy_output ? 1 : 0));
    out += sep; out += (e.strand == strnd::FWD ? '+' : '-');
    out += sep; out += metadata[e.refSeqId].name;
    out += sep; put_int(out, metadata[e.refSeqId].len);
    out += sep; put_int(out, e.refStartPos);
    out += sep; put_int(out, e.refEndPos - (param.legacy_output ? 1 : 0));
    if (!param.legacy_output) {
      out += sep; put_int(out, e.conservedSketches);
      out += sep; put_int(out, e.blockLength);
      out += sep; put_real(out, fakeMapQ);
      out += sep; out += "id:f:"; put_real(out, (param.report_ANI_percentage ? 100.0 : 1.0) * e.nucIdentity);
      out += sep; out += "kc:f:"; put_real(out, e.kmerComplexity);
      if (!param.mergeMappings) { out += sep; out += "jc:f:"; put_real(out, float(e.conservedSketches) / e.sketchSize); }
    } else {
      out += sep; put_real(out, e.nucIdentity * 100.0);
    }
    out += '\n';
  }
}

int64_t MapTail::realTextSelftest(int64_t n, uint64_t seed)
{
  uint64_t x = seed * 0x9E3779B97F4A7C15ULL + 12345;
  auto rnd = [&]() { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
  int64_t bad = 0;
  auto check = [&](auto v) {
    char want[64];
    if (sizeof(v) > sizeof(double)) snprintf(want, sizeof want, "%Lg", (long double)v);
    else snprintf(want, sizeof want, "%g", (double)v);
    std::string got;
    put_real(got, v);
    if (got != want) bad++;
  };
  const double edges[] = {0.0, -0.0, 1.0, 0.1, 0.01, 0.001, 0.0001, 1e-5, 0.5, 0.25, 0.125, 999999.0, 999999.5, 999999.4999, 1e6, 1e7,
                          99999.95, 99999.949, 0.9999995, 0.99999949, 0.00099999949, 0.0009999995, 0.001000001, 255.0, 13.0, 100.0,
                          9.9999995, 123456.5, 12345.65, 1234.565, 0.1234565, 0.01234565, 1e-300, 1e300, -1.5, -0.0625};
  for (double v : edges) {
    check(v); check((float)v); check((long double)v);
    check(std::nextafter(v, 2 * v + 1)); check(std::nextafter(v, -1.0));
    check(std::nextafterf((float)v, 2 * (float)v + 1)); check(std::nextafterf((float)v, -1.0f));
  }
  check(std::numeric_limits<double>::infinity()); check(std::numeric_limits<double>::quiet_NaN());
  for (int64_t i = 0; i < n; i++) {
    const int kind = (int)(rnd() % 8);
    const double u = (double)(rnd() >> 11) / 9007199254740992.0;  // [0, 1)
    double v;
    switch (kind) {
      case 0: v = u; break;
      case 1: v = (float)u; break;
      case 2: v = (double)(rnd() % 4097) / 4096.0; break;                    // dyadic: exact decimal ties
      case 3: v = (double)(rnd() % 2000001) / 2.0; break;                    // halves up to 1e6
      case 4: v = std::pow(10.0, -6.0 + 14.0 * u); break;                    // every magnitude around the fast range
      case 5: v = 100.0 * (double)(float)u; break;                           // identities as percentages
      case 6: v = ((double)(float)u + (double)(float)((double)(rnd() >> 11) / 9007199254740992.0)) / 2.0; break;  // means of floats
      default: v = (double)(rnd() % 1000000) / 100000.0 + ((rnd() & 1) ? 0.000005 : 0.0);  // decimal ties that are not exact in binary
    }
    check(v); check((float)v);
    if ((i & 7) == 0) check((long double)v);
  }
  return bad;
}

void MapTail::formatMappings(const MappingResultsVector_t &readMappings, const std::string &queryName, std::ostream &os) const
{
  std::string text;
  formatMappings(readMappings, queryName, text);
  os << text;
}


}  // namespace skch
