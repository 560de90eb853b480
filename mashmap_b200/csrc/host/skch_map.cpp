#include "skch_map.hpp"
#include <cstdio>
#include <cstdlib>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <limits>
#include <sstream>
#include <thread>
#include <tuple>

#include "../../../include/mashmap_b200_nccl.h"
#include "skch_seqio.hpp"
#include "skch_stats.hpp"

namespace skch {

namespace {

typedef std::chrono::steady_clock Clock;
double since(Clock::time_point t0) { return std::chrono::duration<double>(Clock::now() - t0).count(); }

/* the reference's log lines of an index (winSketch.hpp:228, :403, :418-449) from the statistics of a device build */
void logIndexStats(const Parameters &param, const mm_index_stats &st)
{
  std::cerr << "[mashmap-b200::skch::Sketch::build] minmer windows picked from reference = " << st.n_minmers_before_filter << std::endl;
  std::cerr << "[mashmap-b200::skch::Sketch::index] unique minmers = " << st.n_keys << std::endl;
  if (!st.n_keys) {
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] No minmers." << std::endl;
    return;
  }
  std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] Frequency histogram of minmer interval points = (" << st.hist_min_count << ", "
            << st.hist_min_keys << ") ... (" << st.hist_max_count << ", " << st.hist_max_keys << ")" << std::endl;
  if (st.freq_threshold != std::numeric_limits<int>::max())
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] With threshold " << param.kmer_pct_threshold
              << "%, ignore minmers occurring >= " << st.freq_threshold << " times during lookup." << std::endl;
  else
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] With threshold " << param.kmer_pct_threshold
              << "%, consider all minmers during lookup." << std::endl;
}

[[noreturn]] void die(const std::string &msg)
{
  std::cerr << "[mashmap-b200] ERROR: " << msg << std::endl;
  exit(1);
}

std::string prefix(const std::string &s, const char c) { return s.substr(0, s.find_last_of(c)); }  // computeMap.hpp:1170-1173

}  // namespace

/* ------------------------------------------------------------------------------------------------------ */

void BatchMapper::setRefGroups()
{  // computeMap.hpp:144-161
  refIdGroup.assign(refSketch.metadata.size(), 0);
  if (!param.skip_prefix) return;
  int group = 0;
  size_t start_idx = 0, idx = 0;
  while (start_idx < refSketch.metadata.size()) {
    const auto currPrefix = prefix(refSketch.metadata[start_idx].name, param.prefix_delim);
    idx = start_idx;
    while (idx < refSketch.metadata.size() && currPrefix == prefix(refSketch.metadata[idx].name, param.prefix_delim))
      refIdGroup[idx++] = group;
    group++;
    start_idx = idx;
  }
}

std::string BatchMapper::planShards(const std::vector<uint64_t> &len, const std::vector<int> &group, bool byGroup, int n_shards,
                                    std::vector<int32_t> &first)
{
  const size_t C = len.size();
  std::vector<uint64_t> before(C + 1, 0);  // bases of contigs [0, i)
  for (size_t i = 0; i < C; i++) before[i + 1] = before[i] + len[i];
  std::vector<int32_t> cuts;  // a cut at i: a shard begins with contig i
  for (size_t i = 1; i < C; i++)
    if (!byGroup || group[i] != group[i - 1]) cuts.push_back((int32_t)i);
  if (n_shards < 1) return "--indexShards needs at least one shard";
  if ((size_t)n_shards > cuts.size() + 1)
    return "--indexShards " + std::to_string(n_shards) + ": the reference can be cut in at most " + std::to_string(cuts.size() + 1) +
           " shards (" + std::to_string(cuts.size()) + " possible cut points between " +
           (byGroup ? "runs of contigs in different -Y prefix groups" : "contigs") + ")";
  first.assign(1, 0);
  size_t lo = 0;
  for (int k = 1; k < n_shards; k++) {  // cut k: the allowed point closest to k/N of the bases, leaving one for each later cut
    const double want = (double)before[C] * k / n_shards;
    const size_t hi = cuts.size() - (size_t)(n_shards - 1 - k);
    size_t best = lo;
    for (size_t j = lo; j < hi; j++)
      if (std::abs((double)before[(size_t)cuts[j]] - want) < std::abs((double)before[(size_t)cuts[best]] - want)) best = j;
    first.push_back(cuts[best]);
    lo = best + 1;
  }
  first.push_back((int32_t)C);
  return "";
}

int BatchMapper::getRefGroup(const std::string &seqName) const
{  // computeMap.hpp:164-177
  const auto queryPrefix = prefix(seqName, param.prefix_delim);
  for (size_t i = 0; i < refSketch.metadata.size(); i++)
    if (queryPrefix == prefix(refSketch.metadata[i].name, param.prefix_delim)) return refIdGroup[i];
  return -1;
}

/* Persistent worker threads for the per-read host tail: a part's tail is a few milliseconds of work, creating a hundred
 * threads for it costs as much again. One caller at a time. */
class BatchMapper::WorkerPool {
 public:
  explicit WorkerPool(int n)
  {
    for (int i = 0; i < n; i++) threads_.emplace_back([this, i]() { loop(i); });
  }
  ~WorkerPool()
  {
    { std::lock_guard<std::mutex> lk(mu_); stop_ = true; }
    cvStart_.notify_all();
    for (auto &t : threads_) t.join();
  }
  int size() const { return (int)threads_.size(); }
  /* runs fn() on min(n, size()) workers and returns when all of them are back */
  void run(int n, const std::function<void()> &fn)
  {
    n = std::min(n, size());
    if (n <= 1) { fn(); return; }
    std::unique_lock<std::mutex> lk(mu_);
    fn_ = &fn; want_ = n; done_ = 0; gen_++;
    cvStart_.notify_all();
    cvDone_.wait(lk, [&] { return done_ == want_; });
    fn_ = nullptr;
  }

 private:
  void loop(int idx)
  {
    uint64_t seen = 0;
    while (true) {
      const std::function<void()> *fn = nullptr;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cvStart_.wait(lk, [&] { return stop_ || gen_ != seen; });
        if (stop_) return;
        seen = gen_;
        if (idx < want_) fn = fn_;
      }
      if (fn) {
        (*fn)();
        std::lock_guard<std::mutex> lk(mu_);
        if (++done_ == want_) cvDone_.notify_all();
      }
    }
  }
  std::vector<std::thread> threads_;
  std::mutex mu_;
  std::condition_variable cvStart_, cvDone_;
  const std::function<void()> *fn_ = nullptr;
  uint64_t gen_ = 0;
  int want_ = 0, done_ = 0;
  bool stop_ = false;
};

/* Upload chunks and the L2 phase exclude each other; a waiting L2 phase has priority over the next chunk. */
struct BatchMapper::Gate {
  std::mutex mu;
  std::condition_variable cv;
  int uploading = 0, l2_active = 0, l2_waiting = 0;
};

void BatchMapper::phaseHook(void *user, int phase, int begin)
{
  Gate &g = *static_cast<Gate *>(user);
  std::unique_lock<std::mutex> lk(g.mu);
  if (phase == MM_PHASE_UPLOAD_CHUNK) {
    if (begin) {
      g.cv.wait(lk, [&] { return g.l2_active == 0 && g.l2_waiting == 0; });
      g.uploading++;
    } else {
      g.uploading--;
      g.cv.notify_all();
    }
  } else if (phase == MM_PHASE_L2) {
    if (begin) {
      g.l2_waiting++;
      g.cv.wait(lk, [&] { return g.uploading == 0; });
      g.l2_waiting--;
      g.l2_active++;
    } else {
      g.l2_active--;
      g.cv.notify_all();
    }
  }
}

BatchMapper::BatchMapper(const Parameters &p, const Sketch &refsketch) : param(p), refSketch(refsketch)
{
  // --noSplit (param.split == false): every query is one fragment of its full length (computeMap.hpp:587-607); one longer
  // than a segment is mapped with windowLen = length - segLength (the device's long-fragment path).
  // Map::Map (computeMap.hpp:123-139): setProbs, setRefGroups; plus the per-sketch-size minimum-hit table
  sketchCutoffs = Stat::sketchCutoffs(param.sketchSize, param.kmerSize, param.ANIDiff, param.ANIDiffConf, param.stage1_topANI_filter);
  setRefGroups();
  minHits.assign((size_t)param.sketchSize + 1, 0);
  for (int s = 1; s <= param.sketchSize; s++)
    minHits[s] = Stat::estimateMinimumHitsRelaxed(s, param.kmerSize, param.percentageIdentity, fixed::confidence_interval);
  contigNameId.resize(refSketch.metadata.size());
  for (size_t i = 0; i < refSketch.metadata.size(); i++) {
    auto it = refNameId.find(refSketch.metadata[i].name);
    if (it == refNameId.end()) it = refNameId.emplace(refSketch.metadata[i].name, (int)refNameId.size()).first;
    contigNameId[i] = it->second;
  }
  mm_params mp{};
  mp.kmer_size = param.kmerSize; mp.seg_length = param.segLength; mp.sketch_size = param.sketchSize;
  mp.stage1_topani_filter = param.stage1_topANI_filter; mp.skip_self = param.skip_self;
  mp.skip_prefix = param.skip_prefix; mp.lower_triangular = param.lower_triangular;
  int rc;
  if (param.index_shards > 1) {
    buildShards(mp);
  } else {
    rc = mm_ctx_create(param.device, &mp, &ctx);
    if (rc != MM_OK) die(std::string("mm_ctx_create: ") + mm_last_error(nullptr));
    std::vector<int32_t> clen(refSketch.metadata.size());
    for (size_t i = 0; i < clen.size(); i++) clen[i] = refSketch.metadata[i].len;
    if (refSketch.deviceBuildPending()) {
      // skch::Sketch's build / index / computeFreqHist / dropFreqSeedSet on the device (mm_index_build.cu); with --saveIndex
      // the builder keeps the records before the frequent-seed drop and the lookup, which the files hold
      const bool save = !param.saveIndexFilename.empty();
      mm_index_stats st;
      auto t0 = Clock::now();
      rc = mm_index_build(ctx, refSketch.deviceText(), 0, refSketch.deviceTextOffsets().data(), (int32_t)clen.size(), contigNameId.data(),
                          refIdGroup.data(), param.kmer_pct_threshold, save ? MM_KEEP_LOOKUP | MM_KEEP_UNFILTERED : 0, &st);
      if (rc != MM_OK) die(std::string("mm_index_build: ") + mm_last_error(ctx) + " (--hostIndex builds the index on the host)");
      logIndexStats(param, st);
      std::cerr << "[mashmap-b200::skch::Sketch] index built on the device in " << since(t0) << " s (window scan " << st.ms_scan * 1e-3
                << " s over " << st.n_chunks << " chunks, " << st.n_fixed_chunks << " re-scanned exactly; records " << st.ms_post * 1e-3
                << " s; lookup + frequency filter " << st.ms_lookup * 1e-3 << " s)" << std::endl;
      if (save) refSketch.saveDeviceIndex(ctx, st);
      refSketch.deviceBuildDone(st.freq_threshold);
    } else if (refSketch.deviceLoadPending()) {
      // --loadIndex: Sketch::index / computeFreqHist / dropFreqSeedSet over the file's records on the device; with
      // --saveIndex too, the loaded records and their lookup are written again (winSketch.hpp:122-134 saves after a load)
      const bool save = !param.saveIndexFilename.empty();
      mm_index_stats st;
      auto t0 = Clock::now();
      rc = mm_index_build_minmers(ctx, refSketch.loadedRecords(), refSketch.loadedCount(), 0, clen.data(), contigNameId.data(),
                                  refIdGroup.data(), (int32_t)clen.size(), param.kmer_pct_threshold,
                                  save ? MM_KEEP_LOOKUP | MM_KEEP_UNFILTERED : 0, &st);
      if (rc != MM_OK) die("cannot load index " + refSketch.loadedFile() + ": " + mm_last_error(ctx));
      logIndexStats(param, st);
      std::cerr << "[mashmap-b200::skch::Sketch] index built on the device from the " << refSketch.loadedCount() << " records of "
                << refSketch.loadedFile() << " in " << since(t0) << " s (lookup + frequency filter " << st.ms_lookup * 1e-3 << " s)" << std::endl;
      if (save) refSketch.saveDeviceIndex(ctx, st);
      refSketch.deviceBuildDone(st.freq_threshold);
    } else {
      rc = mm_index_upload(ctx, refSketch.minmerIndex.data(), refSketch.minmerIndex.size(), refSketch.lookupKeys.data(),
                           refSketch.lookupOffsets.data(), refSketch.lookupKeys.size(), refSketch.lookupPoints.data(),
                           refSketch.lookupPoints.size(), refSketch.lookupKeyIsFreq.data(), clen.data(), contigNameId.data(),
                           refIdGroup.data(), (int32_t)clen.size());
      if (rc != MM_OK) die(std::string("mm_index_upload: ") + mm_last_error(ctx));
    }
  }
  for (size_t i = 0; i < std::max<size_t>(1, shards.size()); i++) {
    mm_ctx *c = shards.empty() ? ctx : shards[i].ctx;
    rc = mm_tables_upload(c, sketchCutoffs.data(), (int32_t)sketchCutoffs.size(), minHits.data(), (int32_t)minHits.size());
    if (rc != MM_OK) die(std::string("mm_tables_upload: ") + mm_last_error(c));
  }
  tail_ = new MapTail(param, refSketch.metadata, refIdGroup);
  // one group per device; the first one owns the uploaded image, the others receive a copy over NVLink. A sharded index
  // has one group (the first shard's device): every part runs on all shards
  std::vector<int> devs = param.devices.empty() ? std::vector<int>{param.device} : param.devices;
  if (!shards.empty()) devs.resize(1);
  std::vector<mm_ctx *> others;
  for (size_t d = 0; d < devs.size(); d++) {
    DeviceGroup *g = new DeviceGroup();
    g->device = devs[d];
    if (d == 0) g->owner = ctx;
    else {
      rc = mm_ctx_create(devs[d], &mp, &g->owner);
      if (rc != MM_OK) die(std::string("mm_ctx_create (device ") + std::to_string(devs[d]) + "): " + mm_last_error(nullptr));
      others.push_back(g->owner);
    }
    groups.push_back(g);
  }
  if (!others.empty()) {
    auto t0 = Clock::now();
    rc = mm_index_replicate(ctx, others.data(), (int)others.size());
    if (rc != MM_OK) die(std::string("mm_index_replicate: ") + mm_comm_last_error(nullptr));
    std::cerr << "[mashmap-b200::skch::BatchMapper] index image replicated to " << others.size() << " more device(s) in " << since(t0)
              << " s (one grouped NCCL broadcast)" << std::endl;
  }
  const int G = (int)groups.size();
  for (DeviceGroup *g : groups) {
    // of a device's share of the host threads, three drive its pipeline (upload / kernels / fetch): with CPUs to spare they
    // spin on the device (lowest latency) and the rest run the per-read tail; with eight or fewer threads per device (one
    // process per GPU on a host with few CPUs) they sleep on blocking events instead and every thread runs the tail.
    // Measured per 400 k reads: 2 threads 258 (sleep) vs 507 ms (spin), 8 threads 92 vs 109 ms, 16 threads 110 vs 108 ms.
    const int share = std::max(1, param.threads / G);
    g->blockingWaits = getenv("MM_BLOCKING_WAIT") ? getenv("MM_BLOCKING_WAIT")[0] == '1' : share <= 8;
    g->tailThreads = g->blockingWaits ? share : std::max(1, share - 3);
    if (const char *e = getenv("MM_TAIL_THREADS")) g->tailThreads = std::max(1, atoi(e));  // experiment
    g->tailPool = new WorkerPool(g->tailThreads);
    // further contexts share the device's index image: one lane per pipeline stage in flight (upload / kernels / fetch + tail)
    g->lanes[0].ctx = g->owner;
    g->nLanes = 1;
    const int max_lanes = !shards.empty() ? 1 : getenv("MM_LANES") ? std::max(1, std::min<int>(MAX_LANES, atoi(getenv("MM_LANES")))) : MAX_LANES;  // experiment
    for (int l = 1; l < max_lanes; l++) {
      mm_ctx *c2 = nullptr;
      if (mm_ctx_create(g->device, &mp, &c2) != MM_OK) break;
      if (mm_ctx_share_index(c2, g->owner) != MM_OK) { mm_ctx_destroy(c2); break; }
      g->lanes[l].ctx = c2;
      g->nLanes = l + 1;
    }
    for (int l = 0; l < g->nLanes; l++) mm_ctx_set_wait_mode(g->lanes[l].ctx, g->blockingWaits ? 1 : 0);
    for (auto &sh : shards) mm_ctx_set_wait_mode(sh.ctx, g->blockingWaits ? 1 : 0);
    if (g->nLanes > 1 && !getenv("MM_NO_GATE")) {
      g->gate = new Gate();
      for (int l = 0; l < g->nLanes; l++) mm_ctx_set_phase_hook(g->lanes[l].ctx, &BatchMapper::phaseHook, g->gate);
    }
    if (param.align) g->aligner = new MappingAligner(param, refSketch, g->device);
  }
}

BatchMapper::~BatchMapper()
{
  for (DeviceGroup *g : groups) {
    delete g->tailPool;
    delete g->aligner;
    for (int l = 0; l < MAX_LANES; l++) { g->lanes[l].segRes.release(); g->lanes[l].cands.release(); g->lanes[l].loci.release(); }
    for (int l = g->nLanes - 1; l >= 1; l--) mm_ctx_destroy(g->lanes[l].ctx);
    if (g->owner && g->owner != ctx) mm_ctx_destroy(g->owner);
    delete g->gate;
    delete g;
  }
  delete tail_;
  for (auto &sh : shards)
    if (sh.ctx != ctx) mm_ctx_destroy(sh.ctx);
  if (ctx) mm_ctx_destroy(ctx);
}

/* --indexShards: the plan, pass 1 on every shard (its hashes and their interval-point counts), the frequent seeds of the
 * whole reference on the host, pass 2 (each shard's image with exactly those dropped). The log lines of the index are the
 * unsharded build's. */
void BatchMapper::buildShards(const mm_params &mp)
{
  const int N = param.index_shards;
  const size_t C = refSketch.metadata.size();
  std::vector<uint64_t> len(C);
  for (size_t i = 0; i < C; i++) len[i] = (uint64_t)refSketch.metadata[i].len;
  const std::string why = planShards(len, refIdGroup, param.skip_prefix, N, shardFirst);
  if (!why.empty()) die(why);
  if (!refSketch.deviceBuildPending()) die("--indexShards builds the index on the device");
  const std::vector<int> devs = param.devices.empty() ? std::vector<int>{param.device} : param.devices;
  std::cerr << "[mashmap-b200::skch::BatchMapper] index cut into " << N << " shards by contig:" << std::endl;
  for (int i = 0; i < N; i++) {
    uint64_t bases = 0;
    for (int32_t c = shardFirst[i]; c < shardFirst[i + 1]; c++) bases += len[(size_t)c];
    std::cerr << "[mashmap-b200::skch::BatchMapper]   shard " << i << ": contigs " << shardFirst[i] << "-" << shardFirst[i + 1] - 1 << " ("
              << refSketch.metadata[(size_t)shardFirst[i]].name << " .. " << refSketch.metadata[(size_t)shardFirst[i + 1] - 1].name << "), "
              << bases << " bases, device " << devs[(size_t)i % devs.size()] << std::endl;
  }
  auto t0 = Clock::now();
  shards.resize((size_t)N);
  const char *text = refSketch.deviceText();
  const std::vector<uint64_t> &toff = refSketch.deviceTextOffsets();
  auto shardOffsets = [&](int i) {  // the shard's contigs relative to its first base
    std::vector<uint64_t> o;
    for (int32_t c = shardFirst[i]; c <= shardFirst[i + 1]; c++) o.push_back(toff[(size_t)c] - toff[(size_t)shardFirst[i]]);
    return o;
  };
  std::vector<std::vector<hash_t>> keys((size_t)N);
  std::vector<std::vector<uint32_t>> counts((size_t)N);
  uint64_t picked = 0;
  for (int i = 0; i < N; i++) {
    Shard &sh = shards[(size_t)i];
    const int dev = devs[(size_t)i % devs.size()];
    int rc = mm_ctx_create(dev, &mp, &sh.ctx);
    if (rc != MM_OK) die("mm_ctx_create (device " + std::to_string(dev) + "): " + mm_last_error(nullptr));
    const std::vector<uint64_t> o = shardOffsets(i);
    uint64_t n = 0;
    mm_index_stats st;
    rc = mm_index_key_counts(sh.ctx, text + toff[(size_t)shardFirst[i]], 0, o.data(), (int32_t)(o.size() - 1), nullptr, nullptr, 0, &n, &st);
    if (rc == MM_ECAPACITY) {
      keys[(size_t)i].resize(n);
      counts[(size_t)i].resize(n);
      rc = mm_index_key_counts(sh.ctx, nullptr, 0, nullptr, 0, keys[(size_t)i].data(), counts[(size_t)i].data(), n, &n, nullptr);
    }
    if (rc != MM_OK) die(std::string("mm_index_key_counts (shard ") + std::to_string(i) + "): " + mm_last_error(sh.ctx));
    picked += st.n_minmers_before_filter;
  }
  std::cerr << "[mashmap-b200::skch::Sketch::build] minmer windows picked from reference = " << picked << std::endl;
  std::vector<const hash_t *> kp;
  std::vector<const uint32_t *> cp;
  std::vector<uint64_t> np;
  for (int i = 0; i < N; i++) { kp.push_back(keys[(size_t)i].data()); cp.push_back(counts[(size_t)i].data()); np.push_back(keys[(size_t)i].size()); }
  int threshold = std::numeric_limits<int>::max();
  uint64_t unique = 0;
  const std::vector<hash_t> freq = globalFrequentSeeds(kp, cp, np, param.kmer_pct_threshold, threshold, unique);
  keys.clear(); counts.clear();
  std::vector<int32_t> clen(C);
  for (size_t i = 0; i < C; i++) clen[i] = refSketch.metadata[i].len;
  for (int i = 0; i < N; i++) {
    Shard &sh = shards[(size_t)i];
    const std::vector<uint64_t> o = shardOffsets(i);
    mm_index_stats st;
    int rc = mm_index_build_shard(sh.ctx, text + toff[(size_t)shardFirst[i]], 0, o.data(), shardFirst[i], shardFirst[i + 1] - shardFirst[i],
                                  clen.data(), contigNameId.data(), refIdGroup.data(), (int32_t)C, freq.data(), freq.size(), 0, &st);
    if (rc != MM_OK) die(std::string("mm_index_build_shard (shard ") + std::to_string(i) + "): " + mm_last_error(sh.ctx) +
                         " (a device that cannot hold its shard's image wants more shards)");
    void *blob = nullptr;
    uint64_t bytes = 0;
    mm_index_blob(sh.ctx, &blob, &bytes);
    std::cerr << "[mashmap-b200::skch::BatchMapper]   shard " << i << ": " << st.n_minmers << " minmers, " << st.n_keys << " lookup keys, "
              << bytes << " index bytes" << std::endl;
  }
  std::cerr << "[mashmap-b200::skch::Sketch] index built on the device in " << N << " shards in " << since(t0) << " s" << std::endl;
  refSketch.deviceBuildDone(threshold);
  ctx = shards[0].ctx;
}

/* every shard maps the part. Without -Y one L1 sweep covers all contigs: phase 1 gives each shard's best intersection,
 * phase 2 maps with their maximum and knows which later shards have points (mm_map_resident_with_best). With -Y each
 * prefix group is swept on its own and lies in one shard: every shard's L1 is exact alone. */
void BatchMapper::shardsCompute(Lane &ln)
{
  const bool twoPhase = !param.skip_prefix;
  std::vector<int32_t> best;
  std::vector<uint8_t> after;
  if (twoPhase) {
    best.assign(ln.nseg, 0);
    for (size_t i = 0; i < shards.size(); i++) {
      Shard &sh = shards[i];
      sh.best.resize(ln.nseg);
      if (mm_map_resident_l1_best(sh.ctx, sh.best.data()) != MM_OK)
        die(std::string("mm_map_resident_l1_best (shard ") + std::to_string(i) + "): " + mm_last_error(sh.ctx));
      for (size_t s = 0; s < ln.nseg; s++) best[s] = std::max(best[s], sh.best[s]);
    }
    after.assign(ln.nseg, 0);  // shards from the last one down: does a later one have points of the segment?
  }
  for (size_t i = shards.size(); i-- > 0;) {
    Shard &sh = shards[i];
    const int rc = twoPhase ? mm_map_resident_with_best(sh.ctx, best.data(), after.data(), &sh.nc, &sh.nl) : mm_map_resident(sh.ctx, &sh.nc, &sh.nl);
    if (twoPhase)
      for (size_t s = 0; s < ln.nseg; s++) after[s] |= sh.best[s] > 0 ? 1 : 0;
    if (rc != MM_OK) die(std::string("mm_map_resident (shard ") + std::to_string(i) + "): " + mm_last_error(sh.ctx));
  }
  ln.nc = ln.nl = 0;
  for (const Shard &sh : shards) { ln.nc += sh.nc; ln.nl += sh.nl; }
}

/* the shards' records of each segment, in shard order (= reference order: shards are ascending contig ranges), as one
 * unsharded context returns them */
void BatchMapper::shardsFetch(Lane &ln)
{
  for (size_t i = 0; i < shards.size(); i++) {
    Shard &sh = shards[i];
    sh.segRes.resize(ln.nseg); sh.cands.resize(sh.nc); sh.loci.resize(sh.nl);
    if (mm_batch_fetch(sh.ctx, sh.segRes.data(), sh.cands.data(), sh.nc, sh.loci.data(), sh.nl) != MM_OK)
      die(std::string("mm_batch_fetch (shard ") + std::to_string(i) + "): " + mm_last_error(sh.ctx));
  }
  uint64_t nc = 0, nl = 0;
  for (size_t s = 0; s < ln.nseg; s++) {
    mm_segment_result r = shards[0].segRes[s];
    r.first_candidate = (uint32_t)nc; r.n_candidates = 0; r.n_points = 0; r.best_intersection = 0;
    bool mhTaken = false;
    for (size_t i = 0; i < shards.size(); i++) {
      const mm_segment_result &q = shards[i].segRes[s];
      if (q.sketch_max_hash != r.sketch_max_hash || q.sketch_raw_count != r.sketch_raw_count || q.sketch_size != r.sketch_size)
        die("index shards disagree on the sketch of fragment " + std::to_string(ln.s0 + s) + " (shard " + std::to_string(i) + ")");
      r.n_points += q.n_points;
      r.best_intersection = std::max(r.best_intersection, q.best_intersection);
      // the first reference group in point order decides minimumHits: the first shard with points holds it
      if (!mhTaken && q.n_points > 0) { r.minimum_hits = q.minimum_hits; mhTaken = true; }
      for (uint32_t c = q.first_candidate; c < q.first_candidate + q.n_candidates; c++) {
        mm_l1_candidate cd = shards[i].cands[c];
        memcpy(ln.loci.data() + nl, shards[i].loci.data() + cd.first_locus, (size_t)cd.n_loci * sizeof(mm_l2_locus));
        cd.first_locus = (uint32_t)nl;
        nl += cd.n_loci;
        ln.cands.data()[nc++] = cd;
        r.n_candidates++;
      }
    }
    if (!mhTaken) r.minimum_hits = 0;
    ln.segRes.data()[s] = r;
  }
}

char *BatchMapper::allocBases(uint64_t n_bases)
{
  char *p = nullptr;
  const uint64_t bytes = n_bases / 2 + 256;
  if (mm_host_alloc((void **)&p, bytes) != MM_OK)
    die("cannot allocate the pinned batch buffer (" + std::to_string(bytes >> 20) + " MiB)");
  return p;
}
void BatchMapper::freeBases(char *p) { if (p) mm_host_free(p); }

void BatchMapper::addRead(ReadBatch &b, const std::string &name, const char *seq, offset_t len, seqno_t seqCounter) const
{
  ReadRec rd;
  rd.name = name; rd.len = len; rd.seqCounter = seqCounter; rd.first_seg = b.segs.size();
  rd.refGroup = param.skip_prefix ? getRefGroup(name) : -1;
  int name_id = -1;
  if (param.skip_self) {
    auto it = refNameId.find(name);
    if (it != refNameId.end()) name_id = it->second;
  }
  if (seq) seqio::pack_bases(seq, (uint64_t)len, b.nibbles(b.used));
  auto push = [&](offset_t start, offset_t flen) {
    mm_segment s;
    s.offset = b.used + (uint64_t)start; s.length = flen; s.seq_counter = seqCounter; s.name_id = name_id; s.ref_group = rd.refGroup;
    b.segs.push_back(s);
  };
  if (!param.split && (int64_t)len - param.kmerSize + 1 >= (1LL << 30))
    die("--noSplit: query '" + name + "' (" + std::to_string(len) + " bp) has 2^30 or more k-mer positions: the reference computes "
        "(length - k + 1) * 2 in an int (computeMap.hpp:831), so its result for this query is undefined");
  if (!param.split || len <= param.segLength) push(0, len);  // computeMap.hpp:587-607: one fragment of the whole query
  else {
    const int n = len / param.segLength;  // :610-641
    for (int i = 0; i < n; i++) push(i * param.segLength, param.segLength);
    if (len % param.segLength != 0) push(len - param.segLength, param.segLength);  // :644-671
  }
  rd.n_seg = (uint32_t)(b.segs.size() - rd.first_seg);
  b.used += ((uint64_t)len + ReadBatch::READ_ALIGN - 1) / ReadBatch::READ_ALIGN * ReadBatch::READ_ALIGN;
  b.reads.push_back(std::move(rd));
}

void BatchMapper::finalizeOneToOne(MappingResultsVector_t &allReadMappings, const std::vector<ContigInfo> &qmetadata, std::string &paf) const
{
  tail_->finalizeOneToOne(allReadMappings, qmetadata, paf);
}

void BatchMapper::alignOneToOne(const MappingResultsVector_t &maps, const std::function<const uint8_t *(seqno_t)> &query, std::string &paf)
{
  const size_t n = maps.size(), G = groups.size();
  std::vector<MappingAligner::Item> items(n);
  for (size_t i = 0; i < n; i++) items[i] = {&maps[i], query(maps[i].querySeqId)};
  std::vector<std::vector<std::string>> tags(G);
  auto run = [&](size_t g) {
    const size_t lo = n * g / G, hi = n * (g + 1) / G;
    groups[g]->aligner->align(items.data() + lo, hi - lo, tags[g]);
  };
  std::vector<std::thread> others;
  for (size_t g = 1; g < G; g++) others.emplace_back(run, g);
  run(0);
  for (auto &t : others) t.join();
  std::vector<std::string> all;
  all.reserve(n);
  for (auto &v : tags)
    for (auto &t : v) all.push_back(std::move(t));
  appendTags(paf, all.data());
}

void BatchMapper::reportAlignment() const
{
  uint64_t aligned = 0, tooLong = 0, unaligned = 0, bases = 0;
  double seconds = 0;
  for (const DeviceGroup *g : groups) {
    aligned += g->aligner->aligned; tooLong += g->aligner->tooLong; unaligned += g->aligner->unaligned;
    bases += g->aligner->bases; seconds += g->aligner->seconds;
  }
  std::cerr << "[mashmap-b200::align] " << aligned << " mappings aligned (edlib NW over " << bases << " query + target bases) in "
            << seconds << " s, summed over " << groups.size() << " device(s); " << tooLong
            << " mappings with a region longer than --alignMaxLen " << param.align_max_len << " printed without NM:i / cg:Z";
  if (unaligned) std::cerr << "; " << unaligned << " without an alignment (empty regions)";
  std::cerr << std::endl;
}

/* The three stages of one part (reads [r0, r1) of the batch) on one lane (= one device context with its own stream
 * and buffers). mapBatch runs them as a pipeline: uploads on one thread, kernels on another, fetch + host tail on a
 * third, so that the PCIe copy of part i+1 and the host tail of part i-1 are hidden behind the kernels of part i. */
void BatchMapper::laneUpload(Lane &ln, const ReadBatch &b, size_t r0, size_t r1)
{
  auto t0 = Clock::now();
  ln.r0 = r0; ln.r1 = r1;
  ln.s0 = b.reads[r0].first_seg;
  const size_t s1 = b.reads[r1 - 1].first_seg + b.reads[r1 - 1].n_seg;
  const uint64_t b0 = b.segs[ln.s0].offset;  // a read's first fragment starts at the read's first base (a multiple of READ_ALIGN)
  const uint64_t b1 = r1 < b.reads.size() ? b.segs[b.reads[r1].first_seg].offset : b.used;
  const mm_segment *segp = b.segs.data() + ln.s0;
  if (b0 != 0) {  // fragment offsets are relative to the buffer handed to the device call
    ln.segs.assign(b.segs.begin() + ln.s0, b.segs.begin() + s1);
    for (auto &sg : ln.segs) sg.offset -= b0;
    segp = ln.segs.data();
  }
  ln.nseg = s1 - ln.s0;
  for (size_t i = 0; i < std::max<size_t>(1, shards.size()); i++) {  // a sharded index: the part goes to every shard
    mm_ctx *c = shards.empty() ? ln.ctx : shards[i].ctx;
    const int rc = mm_batch_upload_packed(c, b.nibbles(b0), b1 - b0, segp, ln.nseg);
    if (rc != MM_OK) die(std::string("mm_batch_upload_packed: ") + mm_last_error(c));
  }
  ln.msUpload = since(t0) * 1e3;
  ln.secDevice += since(t0);
}

void BatchMapper::laneCompute(Lane &ln)
{
  auto t0 = Clock::now();
  if (!shards.empty()) {
    shardsCompute(ln);
  } else {
    int rc = mm_map_resident(ln.ctx, &ln.nc, &ln.nl);
    if (rc != MM_OK) die(std::string("mm_map_resident: ") + mm_last_error(ln.ctx));
  }
  ln.msCompute = since(t0) * 1e3;
  ln.secDevice += since(t0);
}

void BatchMapper::laneFinish(DeviceGroup &g, Lane &ln, const ReadBatch &b, std::vector<MappingResultsVector_t> &results,
                             std::vector<std::string> *text, const std::vector<ContigInfo> *qmetadata)
{
  const int tail_threads = g.tailThreads;
  auto t0 = Clock::now();
  const size_t r0 = ln.r0, r1 = ln.r1;
  if (ln.segRes.size() < ln.nseg) ln.segRes.reserve(ln.nseg + ln.nseg / 8 + 1024);
  if (ln.cands.size() < ln.nc) ln.cands.reserve(ln.nc + ln.nc / 8 + 1024);
  if (ln.loci.size() < ln.nl) ln.loci.reserve(ln.nl + ln.nl / 8 + 1024);
  if (!shards.empty()) {
    shardsFetch(ln);
  } else {
    int rc = mm_batch_fetch(ln.ctx, ln.segRes.data(), ln.cands.data(), ln.cands.size(), ln.loci.data(), ln.loci.size());
    if (rc != MM_OK) die(std::string("mm_batch_fetch: ") + mm_last_error(ln.ctx));
  }
  mm_last_stage_ms(ln.ctx, ln.stageMs);
  const double msFetch = since(t0) * 1e3;
  ln.secDevice += since(t0);
  t0 = Clock::now();

  MapTail tail(param, refSketch.metadata, refIdGroup);
  tail.segs = b.segs.data();              // absolute fragment indices (only the lengths are read)
  tail.segRes = ln.segRes.data() - ln.s0; // so that indexing by the absolute fragment index works
  tail.cands = ln.cands.data();
  tail.loci = ln.loci.data();
  tail.qmetadata = qmetadata;
  const size_t nreads = r1 - r0;
  const int nthreads = std::max(1, std::min<int>(tail_threads, (int)((nreads + 255) / 256)));
  std::atomic<size_t> next{r0};
  auto worker = [&]() {
    /* one cache per pool thread, kept across parts and batches: filling its tables costs a binomial search per distinct
     * shared-sketch count (about a millisecond per worker), which every part used to pay again */
    static thread_local IdentityCache idc;
    idc.use(param.kmerSize, param.ANIDiff);
    uint64_t bytes = 0, mapped = 0, maps = 0;
    while (true) {
      const size_t lo = next.fetch_add(256);
      if (lo >= r1) break;
      const size_t hi = std::min(r1, lo + 256);
      for (size_t r = lo; r < hi; r++) {
        results[r].clear();
        if (text) (*text)[r].clear();
        tail.mapRead(b.reads[r], idc, results[r]);
        if (results[r].empty()) continue;
        mapped++;
        maps += results[r].size();
        if (text) {
          tail.formatMappings(results[r], b.reads[r].name, (*text)[r]);
          bytes += (*text)[r].size();
        }
      }
    }
    lastTextBytes += bytes; lastMappedReads += mapped; lastMappings += maps;
  };
  g.tailPool->run(nthreads, worker);
  ln.secTail += since(t0);
  if (text && g.aligner) {  // --align: the part's mappings in output order, then their tags onto the reads' lines
    std::vector<MappingAligner::Item> items;
    for (size_t r = r0; r < r1; r++)
      for (const MappingResult &m : results[r]) items.push_back({&m, b.nibbles(b.segs[b.reads[r].first_seg].offset)});
    std::vector<std::string> tags;
    g.aligner->align(items.data(), items.size(), tags);
    size_t k = 0;
    for (size_t r = r0; r < r1; r++) {
      appendTags((*text)[r], tags.data() + k);
      k += results[r].size();
    }
  }
  static const bool trace = getenv("MM_TRACE") != nullptr;
  if (trace)
    fprintf(stderr, "[trace] lane %d reads %zu-%zu segs %zu: upload %.2f ms (h2d %.2f) compute %.2f ms (kernels %.2f [k1 %.2f k2 %.2f k3 %.2f: prep %.2f scan %.2f]) "
            "fetch %.2f ms (d2h %.2f) tail %.2f ms (%d threads)\n", (int)(&ln - g.lanes), r0, r1, ln.nseg, ln.msUpload, ln.stageMs[3],
            ln.msCompute, ln.stageMs[5], ln.stageMs[0], ln.stageMs[1], ln.stageMs[2], ln.stageMs[6], ln.stageMs[7], msFetch, ln.stageMs[4], since(t0) * 1e3, nthreads);
}

void BatchMapper::mapBatch(const ReadBatch &b, std::vector<MappingResultsVector_t> &results, std::vector<std::string> *text,
                           const std::vector<ContigInfo> *qmetadata)
{
  const size_t nreads = b.reads.size();
  // no up-front clearing: the tail workers reset each read's slot themselves (a million small frees on one thread
  // would cost tens of milliseconds per batch), capacity is reused from the previous batch
  results.resize(nreads);
  if (text) text->resize(nreads);
  lastTextBytes = 0; lastMappedReads = 0; lastMappings = 0;
  if (nreads == 0) return;
  double d0 = 0, t0 = 0;
  for (DeviceGroup *g : groups)
    for (auto &ln : g->lanes) { d0 += ln.secDevice; t0 += ln.secTail; }
  // parts of ~SUB bases (a read is never split across parts)
  // A large batch ends with smaller parts: the last fetch + host tail has nothing left to hide behind. It starts with a
  // half-size part: the kernels wait for the first upload only, and an upload now takes about half as long as the
  // kernels of the same part, so the second (full) part is on the device before the first one's kernels end. (When the
  // upload was barely faster than the kernels, a short first part only made the compute thread wait for the second upload.)
  uint64_t SUB = std::max<uint64_t>(param.sub_batch_bases, 1);
  if (groups.size() > 1)  // several devices: enough parts for every device's three lanes
    SUB = std::max<uint64_t>(std::min<uint64_t>(SUB, b.used / (3 * groups.size()) + 1), (uint64_t)param.segLength);
  std::vector<uint64_t> targets;
  if (b.used >= 4 * SUB) {
    uint64_t left = b.used;
    if (!getenv("MM_NO_RAMP")) { targets.push_back(SUB / 2); left -= SUB / 2; }
    while (left > SUB + SUB / 2 + SUB / 4) { targets.push_back(SUB); left -= SUB; }
    targets.push_back(std::max<uint64_t>(left * 4 / 7, 1));  // the rest in two parts, the last one the smaller
    targets.push_back(~0ULL);
  }
  std::vector<std::pair<size_t, size_t>> parts;
  {
    size_t r0 = 0;
    uint64_t acc = 0;
    for (size_t r = 0; r < nreads; r++) {
      acc += (uint64_t)b.reads[r].len;
      const uint64_t want = parts.size() < targets.size() ? targets[parts.size()] : SUB;
      if (acc >= want || r + 1 == nreads) { parts.emplace_back(r0, r + 1); r0 = r + 1; acc = 0; }
    }
  }
  const size_t G = groups.size();
  if (G == 1) {
    runGroup(*groups[0], b, parts, 0, 1, results, text, qmetadata);
  } else {  // parts dealt round robin to the devices, every device runs its own pipeline
    std::vector<std::thread> drivers;
    for (size_t g = 1; g < G; g++)
      drivers.emplace_back([&, g] { runGroup(*groups[g], b, parts, g, G, results, text, qmetadata); });
    runGroup(*groups[0], b, parts, 0, G, results, text, qmetadata);
    for (auto &t : drivers) t.join();
  }
  memcpy(lastStageMs, groups[0]->lanes[0].stageMs, sizeof(lastStageMs));
  for (DeviceGroup *g : groups)
    for (auto &ln : g->lanes) { secondsDevice += ln.secDevice; secondsHostTail += ln.secTail; }
  secondsDevice -= d0; secondsHostTail -= t0;
}

/* the parts first, first + step, ... of the batch through the three-stage pipeline of one device */
void BatchMapper::runGroup(DeviceGroup &g, const ReadBatch &b, const std::vector<std::pair<size_t, size_t>> &all_parts, size_t first,
                           size_t step, std::vector<MappingResultsVector_t> &results, std::vector<std::string> *text,
                           const std::vector<ContigInfo> *qmetadata)
{
  std::vector<std::pair<size_t, size_t>> parts;
  for (size_t i = first; i < all_parts.size(); i += step) parts.push_back(all_parts[i]);
  const size_t np = parts.size();
  if (np == 0) return;
  Lane *lanes = g.lanes;
  const int nLanes = g.nLanes;
  if (np < 2 || nLanes < 2) {
    for (auto &p : parts) {
      laneUpload(lanes[0], b, p.first, p.second);
      laneCompute(lanes[0]);
      laneFinish(g, lanes[0], b, results, text, qmetadata);
    }
  } else {
    // part i lives on lane i % nLanes; state: 0 waiting, 1 uploaded, 2 computed, 3 finished (its lane is free again)
    const size_t NL = (size_t)nLanes;
    std::vector<int> state(np, 0);
    std::mutex mu;
    std::condition_variable cv;
    auto wait_for = [&](size_t i, int st) {
      std::unique_lock<std::mutex> lk(mu);
      cv.wait(lk, [&] { return state[i] >= st; });
    };
    auto publish = [&](size_t i, int st) {
      { std::lock_guard<std::mutex> lk(mu); state[i] = st; }
      cv.notify_all();
    };
    std::thread uploader([&] {
      for (size_t i = 0; i < np; i++) {
        if (i >= NL) wait_for(i - NL, 3);
        laneUpload(lanes[i % NL], b, parts[i].first, parts[i].second);
        publish(i, 1);
      }
    });
    std::thread finisher([&] {
      for (size_t i = 0; i < np; i++) {
        wait_for(i, 2);
        laneFinish(g, lanes[i % NL], b, results, text, qmetadata);
        publish(i, 3);
      }
    });
    const auto tp0 = Clock::now();
    double waitUpload = 0, tFirst = 0, tLast = 0;
    for (size_t i = 0; i < np; i++) {  // kernels of successive parts run back to back from this thread
      const auto tw = Clock::now();
      wait_for(i, 1);
      waitUpload += since(tw);
      if (i == 0) tFirst = since(tp0);
      laneCompute(lanes[i % NL]);
      publish(i, 2);
    }
    tLast = since(tp0);
    uploader.join();
    finisher.join();
    static const bool trace = getenv("MM_TRACE") != nullptr;
    if (trace)
      fprintf(stderr, "[trace] device %d: %zu parts; first kernels start at %.1f ms, last kernels end at %.1f ms, pipeline drained at %.1f ms; "
              "compute thread waited %.1f ms for uploads\n", g.device, np, tFirst * 1e3, tLast * 1e3, since(tp0) * 1e3, waitUpload * 1e3);
  }
}

/* ------------------------------------------------------------------------------------------------------ */

struct Map::Impl {
  const Parameters &param;
  const Sketch &refSketch;
  PostProcessResultsFn_t processMappingResults;
  Map &self;
  BatchMapper bm;
  std::vector<ContigInfo> qmetadata;  // computeMap.hpp:105 (one-to-one only)
  ReadBatch batch;
  std::ofstream outstrm;
  MappingResultsVector_t allReadMappings;
  seqno_t totalReadsMapped = 0, totalReadsPicked = 0, seqCounter = 0;

  // the batch being filled by the reader (`batch`) and the one being mapped by the worker thread (`inflight`)
  ReadBatch inflight;
  std::thread worker;
  bool workerActive = false;
  std::vector<MappingResultsVector_t> results;
  std::vector<std::string> text;
  std::unique_ptr<seqio::DeviceInflater> inflater;  // BGZF queries, on the run's first device
  std::unique_ptr<seqio::DeviceFastqParser> fastqParser;  // FASTQ queries, on the run's first device

  Impl(const Parameters &p, const Sketch &s, PostProcessResultsFn_t f, Map &m, Clock::time_point tCtor = Clock::now())
      : param(p), refSketch(s), processMappingResults(f), self(m), bm(p, s)
  {
    const double secIndex = since(tCtor);  // the default argument is evaluated before the members are constructed
    auto t1 = Clock::now();
    batch.capacity = param.batch_bases + (uint64_t)param.segLength + 64;
    batch.bases = bm.allocBases(batch.capacity);
    inflight.capacity = batch.capacity;
    inflight.bases = bm.allocBases(inflight.capacity);
    std::cerr << "[mashmap-b200::skch::Map] device contexts + index upload " << secIndex << " s, pinned batch buffers " << since(t1)
              << " s" << std::endl;
  }
  ~Impl()
  {
    waitWorker();
    bm.freeBases(batch.bases);
    bm.freeBases(inflight.bases);
  }

  void waitWorker()
  {
    if (workerActive) { worker.join(); workerActive = false; }
  }

  // --align, -f one-to-one: the nibbles of every mapped query, kept for the run-wide alignment (query id -> offset)
  BigVec<uint8_t> queryNibbles;
  std::vector<uint64_t> queryNibbleAt;

  void keepQueries(const ReadBatch &b)
  {
    for (const ReadRec &rd : b.reads) {
      const uint64_t at = queryNibbles.size(), bytes = ((uint64_t)rd.len + 1) / 2;
      queryNibbles.resize(at + bytes);
      memcpy(queryNibbles.data() + at, b.nibbles(b.segs[rd.first_seg].offset), bytes);
      if (queryNibbleAt.size() <= (size_t)rd.seqCounter) queryNibbleAt.resize((size_t)rd.seqCounter + 1);
      queryNibbleAt[(size_t)rd.seqCounter] = at;
    }
  }

  void mapAndWrite(ReadBatch &b)
  {
    const bool report_now = param.filterMode != filter::ONETOONE;
    if (!report_now && param.align) keepQueries(b);
    bm.mapBatch(b, results, report_now ? &text : nullptr, &qmetadata);
    for (size_t r = 0; r < results.size(); r++) {  // mapModuleHandleOutput (computeMap.hpp:724-747), in input order
      if (!results[r].empty()) totalReadsMapped++;
      if (!report_now) allReadMappings.insert(allReadMappings.end(), results[r].begin(), results[r].end());
      else {
        outstrm << text[r];
        if (processMappingResults != nullptr)
          for (auto &e : results[r]) processMappingResults(e);
      }
    }
    b.clear();
  }

  /* hands the filled batch to the worker thread (mapping + output, in batch order) and goes on reading into the other
   * buffer; one-to-one mode and user callbacks keep the reference's "everything from the calling thread" behaviour */
  void flushBatch()
  {
    if (batch.reads.empty()) return;
    waitWorker();
    std::swap(batch, inflight);
    const bool async = param.filterMode != filter::ONETOONE && processMappingResults == nullptr && !getenv("MM_SERIAL_INPUT");
    if (async) {
      worker = std::thread([this]() { mapAndWrite(inflight); });
      workerActive = true;
    } else {
      mapAndWrite(inflight);
    }
  }

  void onSequence(const std::string &name, const std::string &seq)
  {  // the body of mapQuery's per-sequence callback (computeMap.hpp:317-349)
    const offset_t len = seq.length();
    if (param.filterMode == filter::ONETOONE) qmetadata.push_back(ContigInfo{name, len});
    if (len < param.kmerSize) {
      std::cerr << std::endl << "WARNING, skch::Map::mapQuery, read " << name << " of " << len << "bp "
                << " is not long enough for mapping at segment length " << param.segLength << std::endl;
    } else {
      totalReadsPicked++;
      // a read lives in one batch: flush first if it does not fit in what is left
      if (batch.used + (uint64_t)len > param.batch_bases && !batch.reads.empty()) flushBatch();
      if ((uint64_t)len + 64 > batch.capacity) {  // a single sequence larger than the batch buffer: grow it
        flushBatch();
        bm.freeBases(batch.bases);
        batch.capacity = (uint64_t)len + 64;
        batch.bases = bm.allocBases(batch.capacity);
      }
      bm.addRead(batch, name, seq.data(), len, seqCounter);
      self.totalQueryBases += (uint64_t)len;
    }
    seqCounter++;
  }

  /* onSequence for every record of a window cut by a bulk reader; the bases go straight into the pinned batch buffer,
   * written by all host threads just before the batch is mapped. Src gives size(), name(i), seq_len(i) and pack(i, dst),
   * which writes record i's nibbles to dst. */
  template <class Src>
  void ingestRecords(const Src &src)
  {
    struct CopyJob { size_t rec; uint64_t dst; };
    std::vector<CopyJob> jobs;
    auto runCopies = [&]() {
      if (jobs.empty()) return;
      const int T = std::max(1, std::min<int>(param.threads, (int)(jobs.size() / 16 + 1)));
      std::atomic<size_t> next{0};
      auto worker = [&]() {
        while (true) {
          const size_t b = next.fetch_add(64);
          if (b >= jobs.size()) break;
          const size_t e = std::min(jobs.size(), b + 64);
          for (size_t j = b; j < e; j++) src.pack(jobs[j].rec, batch.nibbles(jobs[j].dst));
        }
      };
      if (T == 1) worker();
      else {
        std::vector<std::thread> pool;
        for (int t = 0; t < T; t++) pool.emplace_back(worker);
        for (auto &th : pool) th.join();
      }
      jobs.clear();
    };
    for (size_t i = 0; i < src.size(); i++) {
      if (src.seq_len(i) > (uint64_t)std::numeric_limits<offset_t>::max()) {
        std::cerr << "[mashmap-b200] ERROR: sequence " << src.name(i) << " is longer than 2^31 bases" << std::endl;
        exit(1);
      }
      const offset_t len = (offset_t)src.seq_len(i);
      const std::string name = src.name(i);
      if (param.filterMode == filter::ONETOONE) qmetadata.push_back(ContigInfo{name, len});
      if (len < param.kmerSize) {
        std::cerr << std::endl << "WARNING, skch::Map::mapQuery, read " << name << " of " << len << "bp "
                  << " is not long enough for mapping at segment length " << param.segLength << std::endl;
      } else {
        totalReadsPicked++;
        if (batch.used + (uint64_t)len > param.batch_bases && !batch.reads.empty()) { runCopies(); flushBatch(); }
        if ((uint64_t)len + 64 > batch.capacity) {
          runCopies();
          flushBatch();
          bm.freeBases(batch.bases);
          batch.capacity = (uint64_t)len + 64;
          batch.bases = bm.allocBases(batch.capacity);
        }
        jobs.push_back(CopyJob{i, batch.used});
        bm.addRead(batch, name, nullptr, len, seqCounter);
        self.totalQueryBases += (uint64_t)len;
      }
      seqCounter++;
    }
    runCopies();
  }

  /* a mapped FASTA file, or one window of an inflated BGZF one: bases packed from the text */
  void ingestMapped(const seqio::FastaText &ff)
  {
    struct Src {
      const seqio::FastaText &ff;
      size_t size() const { return ff.records().size(); }
      std::string name(size_t i) const { return ff.name(ff.records()[i]); }
      uint64_t seq_len(size_t i) const { return ff.records()[i].seq_len; }
      void pack(size_t i, uint8_t *dst) const { ff.pack_bases(ff.records()[i], dst); }
    };
    ingestRecords(Src{ff});
  }

  /* one window of FASTQ records parsed on the device: bases already packed, copied */
  void ingestPacked(const mm_fastq_records &r)
  {
    struct Src {
      const mm_fastq_records &r;
      size_t size() const { return (size_t)r.n_records; }
      std::string name(size_t i) const { return std::string(r.names + r.name_off[i], r.name_off[i + 1] - r.name_off[i]); }
      uint64_t seq_len(size_t i) const { return r.seq_len[i]; }
      void pack(size_t i, uint8_t *dst) const { memcpy(dst, r.nibbles + r.nib_off[i], r.nib_off[i + 1] - r.nib_off[i]); }
    };
    ingestRecords(Src{r});
  }

  void mapQuery()
  {  // computeMap.hpp:263-415
    outstrm.open(param.outFileName);
    auto t0 = Clock::now();
    for (const auto &fileName : param.querySequences) {
      seqio::FastaFile ff;
      if (!getenv("MM_SERIAL_INPUT") && ff.open(fileName, param.threads)) {  // plain FASTA: bulk path
        ingestMapped(ff);
        continue;
      }
      seqio::FastqReader fq;
      if (!getenv("MM_SERIAL_INPUT") && fq.open(fileName)) {  // FASTQ, plain or BGZF: parsed on the device, window by window
        const int dev = param.devices.empty() ? param.device : param.devices[0];
        if (!fastqParser) fastqParser.reset(new seqio::DeviceFastqParser(dev));
        uint64_t windows = 0;
        const int rc = fq.for_each_window(*fastqParser, seqio::fastq_window_bytes(param.batch_bases), param.threads,
                                          [&](const mm_fastq_records &r) { ingestPacked(r); windows++; });
        if (rc < 0) {
          std::cerr << fq.error() << std::endl;
          exit(1);
        }
        std::cerr << "[mashmap-b200::skch::Map::mapQuery] " << fileName << ": FASTQ, parsed on device " << dev << " in "
                  << windows << " windows" << std::endl;
        continue;
      }
      seqio::BgzfFasta bz;
      if (!getenv("MM_SERIAL_INPUT") && bz.open(fileName)) {  // BGZF FASTA: inflated on the device, window by window
        const int dev = param.devices.empty() ? param.device : param.devices[0];
        if (!inflater) inflater.reset(new seqio::DeviceInflater(dev));
        uint64_t windows = 0;
        const int rc = bz.for_each_window(*inflater, seqio::bgzf_window_bytes(param.batch_bases), param.threads,
                                          [&](const seqio::FastaText &t) { ingestMapped(t); windows++; });
        if (rc < 0) {
          std::cerr << bz.error() << std::endl;
          exit(1);
        }
        if (rc == 0) {
          std::cerr << "[mashmap-b200::skch::Map::mapQuery] " << fileName << ": BGZF, inflated on device " << dev << " in "
                    << windows << " windows" << std::endl;
          continue;
        }
      }
      bool ok = seqio::for_each_seq_in_file(fileName, {}, "", [&](const std::string &name, const std::string &seq) { onSequence(name, seq); });
      if (!ok) exit(1);
    }
    const double secRead = since(t0);
    flushBatch();
    waitWorker();
    std::cerr << "[mashmap-b200::skch::Map::mapQuery] input read and handed over in " << secRead << " s, last batch done at "
              << since(t0) << " s" << std::endl;
    self.secondsDevice = bm.secondsDevice;
    self.secondsHostTail = bm.secondsHostTail;
    self.secondsInput = since(t0) - self.secondsDevice - self.secondsHostTail;

    if (param.filterMode == filter::ONETOONE) {  // :358-405
      std::string paf;
      bm.finalizeOneToOne(allReadMappings, qmetadata, paf);
      if (param.align)
        bm.alignOneToOne(allReadMappings, [&](seqno_t id) { return queryNibbles.data() + queryNibbleAt[(size_t)id]; }, paf);
      outstrm << paf;
      if (processMappingResults != nullptr)
        for (auto &e : allReadMappings) processMappingResults(e);
    }
    outstrm.close();
    std::cerr << "[mashmap-b200::skch::Map::mapQuery] count of mapped reads = " << totalReadsMapped
              << ", reads qualified for mapping = " << totalReadsPicked << ", total input reads = " << seqCounter
              << ", total input bp = " << self.totalQueryBases << std::endl;
    if (param.align) bm.reportAlignment();
  }
};

Map::Map(const Parameters &p, const Sketch &refsketch, PostProcessResultsFn_t f) : impl(new Impl(p, refsketch, f, *this))
{
  impl->mapQuery();
}

Map::~Map() { delete impl; }

}  // namespace skch
