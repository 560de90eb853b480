#include "skch_index.hpp"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <numeric>
#include <thread>
#include <tuple>
#include <unordered_set>

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include "../mm_hash.h"
#include "../mm_winmachine.h"
#include "skch_seqio.hpp"

namespace skch {

namespace {

/* getHash of the forward k-mer and of its reverse complement (commonFunc.hpp:138-147, :357-363) for a
 * run-time k: the bytes are packed into 64-bit words exactly as the templated device code does. */
struct HostKmerHasher {
  int k;
  explicit HostKmerHasher(int k_) : k(k_) {}
  static uint64_t murmur(const unsigned char *d, int len)
  { /* MurmurHash3_x64_128 low word, seed 42 (murmur3.h:236-303) */
    const int nblocks = len / 16;
    uint64_t h1 = MM_SEED, h2 = MM_SEED;
    const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
    for (int i = 0; i < nblocks; i++) {
      uint64_t k1, k2;
      memcpy(&k1, d + 16 * i, 8);
      memcpy(&k2, d + 16 * i + 8, 8);
      k1 *= c1; k1 = mm_rotl64(k1, 31); k1 *= c2; h1 ^= k1;
      h1 = mm_rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
      k2 *= c2; k2 = mm_rotl64(k2, 33); k2 *= c1; h2 ^= k2;
      h2 = mm_rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
    }
    const unsigned char *tail = d + nblocks * 16;
    uint64_t k1 = 0, k2 = 0;
    const int tl = len & 15;
    for (int j = tl - 1; j >= 8; j--) k2 |= (uint64_t)tail[j] << (8 * (j - 8));
    if (tl > 8) { k2 *= c2; k2 = mm_rotl64(k2, 33); k2 *= c1; h2 ^= k2; }
    for (int j = std::min(tl, 8) - 1; j >= 0; j--) k1 |= (uint64_t)tail[j] << (8 * j);
    if (tl > 0) { k1 *= c1; k1 = mm_rotl64(k1, 31); k1 *= c2; h1 ^= k1; }
    h1 ^= (uint64_t)len; h2 ^= (uint64_t)len;
    h1 += h2; h2 += h1;
    h1 = mm_fmix64(h1); h2 = mm_fmix64(h2);
    h1 += h2;
    return h1;
  }
};

inline void normalise(char *seq, offset_t len)
{ /* makeUpperCaseAndValidDNA (commonFunc.hpp:97-107) */
  for (offset_t i = 0; i < len; i++) {
    unsigned char c = (unsigned char)seq[i];
    if (c > 96 && c < 123) c -= 32;
    if (!(c == 'A' || c == 'C' || c == 'G' || c == 'T')) c = 'N';
    seq[i] = (char)c;
  }
}

inline MinmerInfo make_mi(hash_t h, offset_t a, offset_t b, seqno_t s, strand_t st)
{
  MinmerInfo m;
  m.hash = h; m.wpos = a; m.wpos_end = b; m.seqId = s; m.strand = st; m._pad = 0;
  return m;
}

/* storage of one window machine on the host */
struct HostMachine {
  wm_machine m;
  std::vector<wm_kmer> ring, heap;
  std::vector<wm_member> mem;
  std::vector<uint64_t> mh;
  std::vector<uint16_t> mslot, sfree;
  std::vector<wm_node> nodes;
  std::vector<wm_record> out;
  HostMachine(int k, int w, int s, size_t out_cap)
      : ring((size_t)wm_ring_cap(w)), heap((size_t)wm_heap_cap(w)), mem((size_t)wm_mem_cap(s)), mh((size_t)wm_mem_cap(s)),
        mslot((size_t)wm_mem_cap(s)), sfree((size_t)wm_mem_cap(s)), nodes((size_t)wm_node_cap(w)), out(out_cap)
  {
    m.ring = ring.data(); m.ring_cap = (int32_t)ring.size();
    m.heap = heap.data(); m.heap_cap = (int32_t)heap.size();
    m.slots = mem.data(); m.mh = mh.data(); m.mslot = mslot.data(); m.sfree = sfree.data(); m.mem_cap = (int32_t)mem.size();
    m.nodes = nodes.data(); m.node_cap = (int32_t)nodes.size();
    m.out = out.data(); m.out_cap = out.size();
    wm_init(m, k, w, s);
  }
};

/* both hashes of the k-mer at position i of the normalised sequence (commonFunc.hpp:357-363) */
inline void kmer_hashes(const char *seq, offset_t i, int k, char *rc, uint64_t &hf, uint64_t &hb)
{
  hf = HostKmerHasher::murmur((const unsigned char *)seq + i, k);
  for (int j = 0; j < k; j++) {  // reverseComplement (commonFunc.hpp:50-73)
    char b = seq[i + j];
    b = b == 'A' ? 'T' : b == 'C' ? 'G' : b == 'G' ? 'C' : b == 'T' ? 'A' : b;
    rc[k - j - 1] = b;
  }
  hb = HostKmerHasher::murmur((const unsigned char *)rc, k);
}

}  // namespace

namespace CommonFunc {

/* the post-processing of addMinmers (commonFunc.hpp:522-568) on the records a window machine emitted, in emission order:
 * malformed-record removal, strand collapse (:534), chunking to <= windowSize (:535-555), sort on (wpos, wpos_end)
 * (:558; std::sort, as the reference: the order of exact ties is libstdc++'s -- or, stable_ties, emission order as the GPU
 * builder keeps it), adjacent (wpos, hash) de-duplication. */
void finishMinmers(std::vector<MinmerInfo> &out, int windowSize, bool stable_ties)
{
  out.erase(std::remove_if(out.begin(), out.end(),
                           [](MinmerInfo &mi) { return mi.wpos < 0 || mi.wpos_end < 0 || mi.wpos == mi.wpos_end; }),
            out.end());
  std::vector<MinmerInfo> chunked;
  for (MinmerInfo &mi : out) {
    mi.strand = mi.strand < 0 ? strnd::REV : strnd::FWD;  // :534 (its AMBIG branch cannot be reached)
    if (mi.wpos_end > mi.wpos + windowSize) {
      const int n = (int)std::ceil(float(mi.wpos_end - mi.wpos) / float(windowSize));
      for (int c = 0; c < n; c++)
        chunked.push_back(make_mi(mi.hash, mi.wpos + c * windowSize, std::min(mi.wpos + c * windowSize + windowSize, mi.wpos_end),
                                  mi.seqId, mi.strand));
    }
  }
  out.erase(std::remove_if(out.begin(), out.end(), [windowSize](MinmerInfo &mi) { return mi.wpos_end - mi.wpos > windowSize; }),
            out.end());
  out.insert(out.end(), chunked.begin(), chunked.end());
  auto before = [](const MinmerInfo &l, const MinmerInfo &r) { return std::tie(l.wpos, l.wpos_end) < std::tie(r.wpos, r.wpos_end); };
  if (stable_ties) std::stable_sort(out.begin(), out.end(), before);  // the device builder's order: exact ties stay in emission order
  else std::sort(out.begin(), out.end(), before);                     // the reference's call; tie order is libstdc++'s
  out.erase(std::unique(out.begin(), out.end(),
                        [](MinmerInfo &l, MinmerInfo &r) { return (l.wpos == r.wpos) && (l.hash == r.hash); }),
            out.end());
}

/*
 * Sliding-window minmer intervals of one contig (commonFunc.hpp:301-570) on the host: the window machine of
 * mm_winmachine.h (the code the GPU builder runs per chunk) driven over the whole contig, then finishMinmers.
 */
void addMinmers(std::vector<MinmerInfo> &out, char *seq, offset_t len, int kmerSize, int windowSize, int alphabetSize,
                int sketchSize, seqno_t seqCounter, bool stable_ties)
{
  normalise(seq, len);
  const offset_t npos = len - kmerSize + 1;
  if (npos <= 0) return;
  HostMachine hm(kmerSize, windowSize, sketchSize, (size_t)npos * 2 + (size_t)sketchSize + 64);
  std::unique_ptr<char[]> rc(new char[kmerSize]);
  for (offset_t i = 0; i < npos; i++) {
    uint64_t hf, hb;
    kmer_hashes(seq, i, kmerSize, rc.get(), hf, hb);
    if (alphabetSize != 4) hb = std::numeric_limits<hash_t>::max();
    wm_step(hm.m, i, hf, hb, seq[i + kmerSize - 1] == 'N');
  }
  wm_flush(hm.m, npos);
  if (hm.m.fail) {
    std::cerr << "[mashmap-b200] ERROR: window machine capacity exceeded on sequence " << seqCounter << std::endl;
    exit(1);
  }
  const size_t base = out.size();
  out.reserve(base + hm.m.out_n);
  std::vector<MinmerInfo> mine;
  mine.reserve(hm.m.out_n);
  for (uint64_t r = 0; r < hm.m.out_n; r++) {
    const wm_record &x = hm.m.out[r];
    mine.push_back(make_mi(x.hash, x.wpos, x.wpos_end, seqCounter, (strand_t)x.votes));
  }
  finishMinmers(mine, windowSize, stable_ties);
  out.insert(out.end(), mine.begin(), mine.end());
}

/*
 * The same contig cut into chunks of `chunk` positions, each scanned by its own machine that starts `warm` positions
 * early from an empty state, and stitched exactly as the GPU builder does (mm_index_build.cu; the scanning routine wm_scan
 * is the very code its kernel runs): a chunk's records that were open at its start take their wpos from the previous
 * chunk's machine; a chunk whose state digest at its start differs from the previous chunk's at its end, or whose refill
 * ever took an expired heap entry, is re-scanned from the previous machine's exact state. Exists so that the stitching
 * logic is tested on the CPU against the unchunked scan. Returns the number of chunks that had to be re-scanned.
 */
template <int K>
static int addMinmersChunkedK(std::vector<MinmerInfo> &out, const uint8_t *seq, offset_t len, int windowSize, int sketchSize,
                              seqno_t seqCounter, offset_t chunk, offset_t warm)
{
  const offset_t npos = len - K + 1;
  if (npos <= 0) return 0;
  std::vector<MinmerInfo> mine;
  const size_t cap = (size_t)(chunk + warm) * 2 + (size_t)sketchSize + 64;
  std::unique_ptr<HostMachine> prev;  // the machine whose state at its end is exact
  wm_kmer_bytes<K> prev_win, cur_win;
  int rescans = 0;
  for (offset_t a = 0; a < npos; a += chunk) {
    const offset_t b = std::min<offset_t>(npos, a + chunk);
    std::unique_ptr<HostMachine> cur(new HostMachine(K, windowSize, sketchSize, cap));
    bool ok = true;
    if (a > 0) {
      const offset_t from = std::max<offset_t>(0, a - warm);
      cur->m.emit_from = a;
      wm_scan<K>(cur->m, cur_win, seq, from, a, true);
      const int32_t wid = a - 1 + K - windowSize;  // the last scanned position's window id
      ok = !cur->m.drained && !cur->m.fail && wm_digest(cur->m, wid) == wm_digest(prev->m, wid);
      cur->m.drained = 0;
      if (ok) {  // inherit the open records' starts
        for (int32_t j = 0; j < cur->m.mem_n; j++) {
          const int32_t pj = wm_find(prev->m, cur->m.mh[j]);
          if (pj >= 0) wm_at(cur->m, j).wpos = wm_at(prev->m, pj).wpos;
        }
      }
    }
    if (ok) {
      wm_scan<K>(cur->m, cur_win, seq, a, b, a == 0);
      if (cur->m.drained && a > 0) ok = false;  // the warm machine's own range touched expired heap entries: not trustworthy
    }
    if (!ok) {  // continue the previous (exact) machine through this chunk instead
      rescans++;
      prev->m.out_n = 0;
      cur = std::move(prev);
      cur_win = prev_win;
      wm_scan<K>(cur->m, cur_win, seq, a, b, false);
    }
    if (b == npos) wm_flush(cur->m, npos);
    if (cur->m.fail) { std::cerr << "[mashmap-b200] ERROR: window machine capacity exceeded" << std::endl; exit(1); }
    for (uint64_t r = 0; r < cur->m.out_n; r++) {
      const wm_record &x = cur->m.out[r];
      mine.push_back(make_mi(x.hash, x.wpos, x.wpos_end, seqCounter, (strand_t)x.votes));
    }
    cur->m.out_n = 0;
    prev = std::move(cur);
    prev_win = cur_win;
  }
  finishMinmers(mine, windowSize, false);
  out.insert(out.end(), mine.begin(), mine.end());
  return rescans;
}

int addMinmersChunked(std::vector<MinmerInfo> &out, char *seq, offset_t len, int kmerSize, int windowSize, int sketchSize,
                      seqno_t seqCounter, offset_t chunk, offset_t warm)
{
  switch (kmerSize) {
#define X(KK) case KK: return addMinmersChunkedK<KK>(out, (const uint8_t *)seq, len, windowSize, sketchSize, seqCounter, chunk, warm);
    X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16) X(17) X(18) X(19) X(20) X(21) X(22) X(23) X(24) X(25) X(26) X(27)
    X(28) X(29) X(30) X(31) X(32)
#undef X
    default: std::cerr << "[mashmap-b200] ERROR: k-mer size " << kmerSize << " is outside 8..32" << std::endl; exit(1);
  }
}

uint64_t getReferenceSize(const std::vector<std::string> &refSequences)
{
  uint64_t count = 0;
  for (auto &f : refSequences) {
    std::ifstream in(f, std::ifstream::ate | std::ifstream::binary);
    count += (uint64_t)(in.tellg());
  }
  return count;
}

}  // namespace CommonFunc

/* The limits of the B200 path, checked BEFORE the reference is read and indexed (the reference itself accepts these
 * inputs; failing after a 3 Gbp index has been built would waste minutes): see README.md, "Limits". */
static void checkPathLimits(const Parameters &p)
{
  auto die = [](const std::string &m) { std::cerr << "[mashmap-b200] ERROR: " << m << std::endl; exit(1); };
  mm_params mp{};
  mp.kmer_size = p.kmerSize; mp.seg_length = p.segLength; mp.sketch_size = std::max(1, p.sketchSize);
  if (mm_params_check(&mp) != MM_OK) die(mm_last_error(nullptr));
  if (p.sketchSize > 1000)
    std::cerr << "[mashmap-b200] NOTE: sketch size " << p.sketchSize << " > 1000: the L2 stage uses its general kernel (about 4x slower)" << std::endl;
}

Sketch::Sketch(const Parameters &p) : param(p)
{
  checkPathLimits(param);
  build();
  if (!deviceBuildPending() && !deviceLoadPending()) finish();
}

Sketch::~Sketch()
{
  free(deviceText_);
  if (loaded_) mm_host_free(loaded_);
}

void Sketch::deviceBuildDone(int freq_threshold) const
{
  free(deviceText_);
  deviceText_ = nullptr;
  deviceTextOffsets_.clear();
  if (loaded_) mm_host_free(loaded_);
  loaded_ = nullptr;
  freqThreshold = freq_threshold;
}

void Sketch::saveDeviceIndex(mm_ctx *ctx, const mm_index_stats &st) const
{
  auto t0 = std::chrono::steady_clock::now();
  BigVec<MinmerInfo> mi(st.n_minmers_before_filter);
  BigVec<hash_t> keys(st.n_keys);
  BigVec<uint64_t> offsets(st.n_keys + 1, 0);
  BigVec<IntervalPoint> points(st.n_points);
  uint64_t n = 0;
  int rc = mm_index_download_unfiltered(ctx, mi.data(), mi.size(), &n);
  if (rc == MM_OK && st.n_keys) rc = mm_index_download(ctx, nullptr, keys.data(), offsets.data(), points.data(), nullptr);
  if (rc == MM_OK) rc = mm_index_release_kept(ctx);  // before the batch buffers are sized: mapping sees the memory of a run without --saveIndex
  if (rc != MM_OK) {
    std::cerr << "[mashmap-b200::skch::Sketch] ERROR: cannot download the index to save it: " << mm_last_error(ctx) << std::endl;
    exit(1);
  }
  writeIndexFiles(mi.data(), n, keys.data(), offsets.data(), points.data(), keys.size());
  std::cerr << "[mashmap-b200::skch::Sketch] index saved to " << param.saveIndexFilename << " in "
            << std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() << " s" << std::endl;
}

Sketch::Sketch(const Parameters &p, const std::vector<ContigInfo> &contigs, const std::vector<const char *> &seqs)
    : metadata(contigs), param(p)
{
  sequencesByFileInfo.push_back((int)contigs.size());
  if (param.align)
    for (size_t i = 0; i < seqs.size(); i++) keepForAlign(seqs[i], (size_t)metadata[i].len);
  buildFromMemory(seqs);
  finish();
}

void Sketch::keepForAlign(const char *seq, size_t len)
{
  const uint64_t at = refNibbles_.size();
  refNibbleOffsets_.push_back(at);
  refNibbles_.resize(at + (len + 1) / 2);
  seqio::pack_bases(seq, len, refNibbles_.data() + at);
}

Sketch::Sketch(const Parameters &p, const std::vector<ContigInfo> &contigs, MI_Type &&minmers)
    : metadata(contigs), minmerIndex(std::move(minmers)), param(p)
{
  sequencesByFileInfo.push_back((int)contigs.size());
  finish();
}

void Sketch::buildFromMemory(const std::vector<const char *> &seqs)
{
  auto tb0 = std::chrono::steady_clock::now();
  std::vector<MI_Type> outputs(seqs.size());
  std::atomic<size_t> next{0};
  const int nthreads = std::max(1, param.threads);
  std::vector<std::thread> pool;
  for (int t = 0; t < nthreads; t++) {
    pool.emplace_back([&]() {
      while (true) {
        const size_t i = next.fetch_add(1);
        if (i >= seqs.size()) break;
        const offset_t len = metadata[i].len;
        if (len < param.kmerSize) continue;
        std::string buf(seqs[i], (size_t)len);  // addMinmers normalises in place
        CommonFunc::addMinmers(outputs[i], &buf[0], len, param.kmerSize, param.segLength, param.alphabetSize,
                               param.sketchSize, (seqno_t)i);
      }
    });
  }
  for (auto &th : pool) th.join();
  std::cerr << "[mashmap-b200::skch::Sketch] minmer windows computed in "
            << std::chrono::duration<double>(std::chrono::steady_clock::now() - tb0).count() << " s" << std::endl;
  size_t total = 0;
  for (auto &o : outputs) total += o.size();
  minmerIndex.reserve(total);
  for (auto &o : outputs) {
    minmerIndex.insert(minmerIndex.end(), o.begin(), o.end());
    MI_Type().swap(o);
  }
  std::cerr << "[mashmap-b200::skch::Sketch::build] minmer windows picked from reference = " << minmerIndex.size() << std::endl;
}

void Sketch::finish()
{
  auto t0 = std::chrono::steady_clock::now();
  if (!param.saveIndexFilename.empty()) {  // winSketch.hpp:127-134: saved BEFORE frequent seeds are dropped
    saving_ = true;
    index();
    saving_ = false;
    writeIndexFiles(minmerIndex.data(), minmerIndex.size(), lookupKeys.data(), lookupOffsets.data(), lookupPoints.data(), lookupKeys.size());
  }
  index();
  std::cerr << "[mashmap-b200::skch::Sketch] lookup index + frequency filter in "
            << std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() << " s" << std::endl;
}

void Sketch::build()
{  // winSketch.hpp:147-230
  std::unordered_set<std::string> allowed;
  if (!param.target_list.empty()) {
    std::ifstream fl(param.target_list);
    std::string name;
    while (getline(fl, name)) allowed.insert(name);
  }
  // the device builds the index unless --hostIndex asks for the host: from the text, or from the records of --loadIndex
  const bool device = !param.host_index && param.kmerSize >= 8 && param.kmerSize <= 32;
  const bool on_device = device && param.loadIndexFilename.empty();
  if (!param.loadIndexFilename.empty()) {
    bool ok = device ? loadIndexForDevice()
                     : param.loadIndexFilename.extension() == ".tsv" ? loadIndexTSV(param.loadIndexFilename.string())
                                                                     : loadIndexBinary(param.loadIndexFilename.string());
    if (!ok) {
      std::cerr << "[mashmap-b200::skch::Sketch::build] ERROR: cannot load index " << param.loadIndexFilename << std::endl;
      exit(1);
    }
  }
  // contigs are read by this thread and sketched by a pool; outputs are appended in input order
  struct Task { std::string seq; seqno_t id; };
  std::vector<std::unique_ptr<Task>> tasks;
  seqno_t seqCounter = 0;
  uint64_t textBytes = 0, textCap = 0;
  if (on_device) deviceTextOffsets_.push_back(0);
  auto onSequence = [&](const std::string &name, const std::string &seq) {
    offset_t len = seq.length();
    metadata.push_back(ContigInfo{name, len});
    if (param.align) keepForAlign(seq.data(), seq.size());
    if (on_device) {  // every contig, also the short ones: seqId = position in metadata
      if (textBytes + seq.size() + 64 > textCap) {
        textCap = std::max<uint64_t>(textCap * 2, textBytes + seq.size() + (64ULL << 20));
        deviceText_ = (char *)realloc(deviceText_, textCap);
        if (!deviceText_) { std::cerr << "[mashmap-b200] ERROR: out of memory reading the reference" << std::endl; exit(1); }
      }
      memcpy(deviceText_ + textBytes, seq.data(), seq.size());
      textBytes += seq.size();
      deviceTextOffsets_.push_back(textBytes);
    } else if (len >= param.kmerSize && param.loadIndexFilename.empty()) {
      tasks.emplace_back(new Task{seq, seqCounter});
    }
    seqCounter++;
  };
  std::unique_ptr<seqio::DeviceInflater> inflater;  // BGZF references of an index built on the device
  for (const auto &fileName : param.refSequences) {
    seqio::BgzfFasta bz;
    int rc = 1;
    if (on_device && !getenv("MM_SERIAL_INPUT") && bz.open(fileName)) {
      const int dev = param.devices.empty() ? param.device : param.devices[0];
      if (!inflater) inflater.reset(new seqio::DeviceInflater(dev));
      std::string seq;
      uint64_t windows = 0;
      // the line reader's semantics: a record outside --targetPrefix / --targetList comes with an empty sequence
      rc = bz.for_each_window(*inflater, seqio::bgzf_window_bytes(param.batch_bases), param.threads, [&](const seqio::FastaText &t) {
        for (const seqio::FastaRecord &r : t.records()) {
          const std::string name = t.name(r);
          const bool keep = (param.target_prefix.empty() || name.compare(0, param.target_prefix.length(), param.target_prefix) == 0) &&
                            (allowed.empty() || allowed.count(name));
          seq.resize(keep ? r.seq_len : 0);
          if (keep) t.copy_bases(r, &seq[0]);
          onSequence(name, seq);
        }
        windows++;
      });
      if (rc < 0) {
        std::cerr << bz.error() << std::endl;
        exit(1);
      }
      if (rc == 0)
        std::cerr << "[mashmap-b200::skch::Sketch::build] " << fileName << ": BGZF, inflated on device " << dev << " in "
                  << windows << " windows" << std::endl;
    }
    if (rc == 1 && !seqio::for_each_seq_in_file(fileName, allowed, param.target_prefix, onSequence)) exit(1);
    sequencesByFileInfo.push_back(seqCounter);
  }
  if (seqCounter == 0) {
    std::cerr << "[mashmap-b200::skch::Sketch::build] ERROR: No sequences indexed!" << std::endl;
    exit(1);
  }
  if (on_device) {
    if (!deviceText_) deviceText_ = (char *)malloc(64);  // only empty contigs: still "pending", the device reports an empty index
    return;
  }
  if (deviceLoadPending()) return;
  if (param.loadIndexFilename.empty()) {
    std::vector<MI_Type> outputs(tasks.size());
    std::atomic<size_t> next{0};
    const int nthreads = std::max(1, param.threads);
    std::vector<std::thread> pool;
    for (int t = 0; t < nthreads; t++) {
      pool.emplace_back([&]() {
        while (true) {
          const size_t i = next.fetch_add(1);
          if (i >= tasks.size()) break;
          Task &tk = *tasks[i];
          CommonFunc::addMinmers(outputs[i], &tk.seq[0], (offset_t)tk.seq.size(), param.kmerSize, param.segLength,
                                 param.alphabetSize, param.sketchSize, tk.id);
          std::string().swap(tk.seq);
        }
      });
    }
    for (auto &th : pool) th.join();
    size_t total = 0;
    for (auto &o : outputs) total += o.size();
    minmerIndex.reserve(total);
    for (auto &o : outputs) {
      minmerIndex.insert(minmerIndex.end(), o.begin(), o.end());
      MI_Type().swap(o);
    }
  }
  std::cerr << "[mashmap-b200::skch::Sketch::build] minmer windows picked from reference = " << minmerIndex.size() << std::endl;
}

/*
 * index() + computeFreqHist() + computeFreqSeedSet() + dropFreqSeedSet() of the reference
 * (winSketch.hpp:379-453, :488-504), producing the flattened lookup (keys ascending) and dropping the frequent
 * hashes from minmerIndex -- done in one parallel pass structure instead of a hash map of vectors:
 *   1. partition the entries by hash range (sampled splitters) keeping index order inside each part,
 *   2. per part (one thread each): stable sort by hash, then per hash emit OPEN/CLOSE points in index order,
 *      fusing an interval that starts where the previous one of the same hash closed (:388-396),
 *   3. histogram of points per hash -> freqThreshold (:415-441),
 *   4. per part: flag the entries of frequent hashes; compact minmerIndex (:497-504).
 */
void Sketch::index()
{
  static const bool trace = getenv("MM_TRACE") != nullptr;
  auto tph = std::chrono::steady_clock::now();
  auto phase = [&](const char *what) {
    if (trace) std::cerr << "[trace] Sketch::index " << what << ": "
                         << std::chrono::duration<double>(std::chrono::steady_clock::now() - tph).count() << " s" << std::endl;
    tph = std::chrono::steady_clock::now();
  };
  const size_t n = minmerIndex.size();
  lookupKeys.clear(); lookupOffsets.clear(); lookupPoints.clear(); lookupKeyIsFreq.clear();
  const int T = std::max(1, std::min(param.threads, 256));
  const size_t P = (size_t)T * 4; /* parts */
  std::vector<hash_t> splitters;
  if (n > 0 && P > 1) {
    const size_t ns = std::min<size_t>(n, 1 << 16);
    std::vector<hash_t> sample(ns);
    for (size_t i = 0; i < ns; i++) sample[i] = minmerIndex[(size_t)((double)i * n / ns)].hash;
    std::sort(sample.begin(), sample.end());
    for (size_t p = 1; p < P; p++) splitters.push_back(sample[p * ns / P]);
  }
  auto part_of = [&](hash_t h) { return (size_t)(std::upper_bound(splitters.begin(), splitters.end(), h) - splitters.begin()); };
  const size_t NP = splitters.size() + 1;
  auto run_threads = [&](size_t n_tasks, const std::function<void(size_t)> &fn) {
    std::atomic<size_t> next{0};
    std::vector<std::thread> pool;
    const int nt = (int)std::min<size_t>((size_t)T, std::max<size_t>(n_tasks, 1));
    for (int t = 0; t < nt; t++)
      pool.emplace_back([&]() {
        while (true) {
          const size_t i = next.fetch_add(1);
          if (i >= n_tasks) break;
          fn(i);
        }
      });
    for (auto &th : pool) th.join();
  };
  /* Fresh memory is the expensive resource here (first touch of a page costs far more than copying it), so the pass
   * allocates each big array once: one (hash, position) pair per entry, and the final arrays. */
  /* 1. counting partition into (hash, index position) pairs: chunk c of the entries x part p */
  const size_t C = (size_t)T;
  const size_t chunk = (n + C - 1) / std::max<size_t>(C, 1);
  std::vector<std::vector<uint64_t>> at(C, std::vector<uint64_t>(NP, 0));
  run_threads(C, [&](size_t c) {
    const size_t lo = std::min(n, c * chunk), hi = std::min(n, lo + chunk);
    for (size_t i = lo; i < hi; i++) at[c][part_of(minmerIndex[i].hash)]++;
  });
  std::vector<uint64_t> part_start(NP + 1, 0);
  {
    uint64_t run = 0;
    for (size_t p = 0; p < NP; p++) {
      part_start[p] = run;
      for (size_t c = 0; c < C; c++) { const uint64_t k = at[c][p]; at[c][p] = run; run += k; }
    }
    part_start[NP] = run;
  }
  typedef std::pair<hash_t, uint64_t> HashPos;
  BigVec<HashPos> kv(n);
  run_threads(C, [&](size_t c) {
    const size_t lo = std::min(n, c * chunk), hi = std::min(n, lo + chunk);
    std::vector<uint64_t> &pos = at[c];
    for (size_t i = lo; i < hi; i++) {
      const hash_t h = minmerIndex[i].hash;
      kv[pos[part_of(h)]++] = HashPos(h, (uint64_t)i);
    }
  });
  phase("partition");
  /* 2. per part: order by (hash, index position) and count keys and interval points (winSketch.hpp:383-396: an interval
   *    that starts where the previous one of the same hash ended is fused into it -- whatever the contig) */
  std::vector<uint64_t> n_keys(NP + 1, 0), n_pts(NP + 1, 0);
  run_threads(NP, [&](size_t p) {
    HashPos *b = kv.data() + part_start[p], *e = kv.data() + part_start[p + 1];
    std::sort(b, e);
    uint64_t keys = 0, pts = 0;
    for (HashPos *it = b; it != e;) {
      const hash_t h = it->first;
      bool have = false;
      offset_t last_pos = 0;
      for (; it != e && it->first == h; ++it) {
        const MinmerInfo &mi = minmerIndex[it->second];
        if (!have || last_pos != mi.wpos) pts += 2;
        have = true;
        last_pos = mi.wpos_end;
      }
      keys++;
    }
    n_keys[p + 1] = keys; n_pts[p + 1] = pts;
  });
  for (size_t p = 0; p < NP; p++) { n_keys[p + 1] += n_keys[p]; n_pts[p + 1] += n_pts[p]; }
  phase("per-part sort + count");
  /* 3. emit straight into the final arrays (parts are ascending hash ranges) */
  lookupKeys.resize(n_keys[NP]);
  lookupOffsets.resize(n_keys[NP] + 1);
  lookupPoints.resize(n_pts[NP]);
  lookupKeyIsFreq.resize(n_keys[NP]);
  run_threads(NP, [&](size_t p) {
    const HashPos *b = kv.data() + part_start[p], *e = kv.data() + part_start[p + 1];
    uint64_t k = n_keys[p], w = n_pts[p];
    for (const HashPos *it = b; it != e;) {
      const hash_t h = it->first;
      const uint64_t first_pt = w;
      for (; it != e && it->first == h; ++it) {
        const MinmerInfo &mi = minmerIndex[it->second];
        if (w == first_pt || lookupPoints[w - 1].pos != mi.wpos) {
          IntervalPoint a{}; a.pos = mi.wpos; a.hash = mi.hash; a.seqId = mi.seqId; a.side = side::OPEN;
          IntervalPoint c2{}; c2.pos = mi.wpos_end; c2.hash = mi.hash; c2.seqId = mi.seqId; c2.side = side::CLOSE;
          lookupPoints[w++] = a;
          lookupPoints[w++] = c2;
        } else {
          lookupPoints[w - 1].pos = mi.wpos_end;
        }
      }
      lookupKeys[k] = h;
      lookupOffsets[k] = first_pt;
      lookupKeyIsFreq[k] = 0;
      k++;
    }
  });
  lookupOffsets[n_keys[NP]] = n_pts[NP];
  phase("emit keys / points");
  std::cerr << "[mashmap-b200::skch::Sketch::index] unique minmers = " << lookupKeys.size() << std::endl;
  if (saving_) return; /* the caller saves the un-filtered index first (winSketch.hpp:127-134) and calls again */

  /* 4. frequency threshold (winSketch.hpp:410-453) */
  if (lookupKeys.empty()) {
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] No minmers." << std::endl;
    return;
  }
  std::map<int, int> hist;
  {  // per-part counts first (one map update per key on one thread cost seconds at 140 M keys)
    std::vector<std::vector<uint32_t>> ph(NP);
    run_threads(NP, [&](size_t p) {
      std::vector<uint32_t> &hh = ph[p];
      for (uint64_t k = n_keys[p]; k < n_keys[p + 1]; k++) {
        const uint64_t c = lookupOffsets[k + 1] - lookupOffsets[k];
        if (c >= hh.size()) hh.resize((size_t)c + 1, 0);
        hh[c]++;
      }
    });
    for (size_t p = 0; p < NP; p++)
      for (size_t c = 0; c < ph[p].size(); c++)
        if (ph[p][c]) hist[(int)c] += (int)ph[p][c];
  }
  freqThreshold = computeFreqThreshold(hist, (int64_t)lookupKeys.size(), param.kmer_pct_threshold);
  phase("histogram");
  /* 5. frequent seeds (:488-504): flag the keys, drop their entries from minmerIndex only */
  if (freqThreshold == std::numeric_limits<int>::max()) return;
  std::vector<std::vector<uint64_t>> dropped(NP); /* index positions to remove (few: 0.001 % of the keys by default) */
  run_threads(NP, [&](size_t p) {
    const HashPos *it = kv.data() + part_start[p];
    for (uint64_t k = n_keys[p]; k < n_keys[p + 1]; k++) {
      const hash_t h = lookupKeys[k];
      const bool fr = (int64_t)(lookupOffsets[k + 1] - lookupOffsets[k]) >= (int64_t)freqThreshold;
      if (fr) lookupKeyIsFreq[k] = 1;
      for (; it != kv.data() + part_start[p + 1] && it->first == h; ++it)
        if (fr) dropped[p].push_back(it->second);
    }
  });
  std::vector<uint64_t> drop;
  for (auto &d : dropped) drop.insert(drop.end(), d.begin(), d.end());
  phase("frequent flags");
  if (!drop.empty()) {  // order-preserving removal in place: the runs between removed entries slide down
    std::sort(drop.begin(), drop.end());
    size_t w = drop[0];
    for (size_t j = 0; j < drop.size(); j++) {
      const size_t from = drop[j] + 1, to = j + 1 < drop.size() ? drop[j + 1] : n;
      if (to > from) memmove(&minmerIndex[w], &minmerIndex[from], (to - from) * sizeof(MinmerInfo));
      w += to - from;
    }
    minmerIndex.resize(w);
  }
  phase("compaction");
}

int computeFreqThreshold(const std::map<int, int> &hist, int64_t totalUniqueMinmers, float kmer_pct_threshold)
{  // winSketch.hpp:418-449
  std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] Frequency histogram of minmer interval points = ("
            << hist.begin()->first << ", " << hist.begin()->second << ") ... (" << hist.rbegin()->first << ", "
            << hist.rbegin()->second << ")" << std::endl;
  int freqThreshold = std::numeric_limits<int>::max();
  int64_t minmerToIgnore = totalUniqueMinmers * kmer_pct_threshold / 100;
  int64_t sum = 0;
  for (auto it = hist.rbegin(); it != hist.rend(); it++) {
    sum += it->second;
    if (sum < minmerToIgnore) {
      freqThreshold = it->first;
    } else if (sum == minmerToIgnore) {
      freqThreshold = it->first;
      break;
    } else {
      break;
    }
  }
  if (freqThreshold != std::numeric_limits<int>::max())
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] With threshold " << kmer_pct_threshold
              << "%, ignore minmers occurring >= " << freqThreshold << " times during lookup." << std::endl;
  else
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] With threshold " << kmer_pct_threshold
              << "%, consider all minmers during lookup." << std::endl;
  return freqThreshold;
}

std::vector<hash_t> globalFrequentSeeds(const std::vector<const hash_t *> &keys, const std::vector<const uint32_t *> &counts,
                                        const std::vector<uint64_t> &n, float kmer_pct_threshold, int &threshold, uint64_t &n_unique)
{
  /* one pass of an N-way merge (N is small) gives the union's distinct hashes with their summed counts */
  const size_t N = keys.size();
  std::vector<uint64_t> at(N, 0);
  std::vector<std::pair<hash_t, uint32_t>> merged;
  uint64_t total = 0;
  for (size_t i = 0; i < N; i++) total += n[i];
  merged.reserve(total);
  while (true) {
    bool any = false;
    hash_t h = 0;
    for (size_t i = 0; i < N; i++)
      if (at[i] < n[i] && (!any || keys[i][at[i]] < h)) { h = keys[i][at[i]]; any = true; }
    if (!any) break;
    uint64_t c = 0;
    for (size_t i = 0; i < N; i++)
      if (at[i] < n[i] && keys[i][at[i]] == h) c += counts[i][at[i]++];
    merged.emplace_back(h, (uint32_t)std::min<uint64_t>(c, std::numeric_limits<uint32_t>::max()));
  }
  n_unique = merged.size();
  std::cerr << "[mashmap-b200::skch::Sketch::index] unique minmers = " << n_unique << std::endl;
  threshold = std::numeric_limits<int>::max();
  std::vector<hash_t> freq;
  if (merged.empty()) {
    std::cerr << "[mashmap-b200::skch::Sketch::computeFreqHist] No minmers." << std::endl;
    return freq;
  }
  std::map<int, int> hist;
  for (const auto &e : merged) hist[(int)e.second]++;
  threshold = computeFreqThreshold(hist, (int64_t)merged.size(), kmer_pct_threshold);
  if (threshold == std::numeric_limits<int>::max()) return freq;
  for (const auto &e : merged)
    if ((int64_t)e.second >= (int64_t)threshold) freq.push_back(e.first);  // isFreqSeed: count >= threshold (:488-495)
  return freq;
}

void Sketch::writeIndexFiles(const MinmerInfo *mi, size_t n, const hash_t *keys, const uint64_t *offsets, const IntervalPoint *points,
                             size_t n_keys) const
{
  const std::string path = param.saveIndexFilename.string();
  if (param.saveIndexFilename.extension() == ".tsv") saveIndexTSV(path, mi, n);
  else saveIndexBinary(path, mi, n);
  savePosListBinary(path, keys, offsets, points, n_keys);
}

void Sketch::saveIndexTSV(const std::string &path, const MinmerInfo *records, size_t n)
{  // winSketch.hpp:270-279
  std::ofstream o(path);
  o << "seqId" << "\t" << "strand" << "\t" << "start" << "\t" << "end" << "\t" << "hash\n";
  for (size_t i = 0; i < n; i++) {
    const MinmerInfo &mi = records[i];
    o << mi.seqId << "\t" << std::to_string(mi.strand) << "\t" << mi.wpos << "\t" << mi.wpos_end << "\t" << mi.hash << "\n";
  }
}

void Sketch::saveIndexBinary(const std::string &prefix, const MinmerInfo *records, size_t n)
{  // winSketch.hpp:284-293
  std::ofstream o(prefix + ".index", std::ios::binary);
  size_t size = n;
  o.write((const char *)&size, sizeof(size));
  o.write((const char *)records, size * sizeof(MinmerInfo));
}

void Sketch::savePosListBinary(const std::string &prefix, const hash_t *keys, const uint64_t *offsets, const IntervalPoint *points,
                               size_t n_keys)
{  // winSketch.hpp:298-315 (key order is unspecified in the reference's hash map; ascending here)
  std::ofstream o(prefix + ".map", std::ios::binary);
  size_t size = n_keys;
  o.write((const char *)&size, sizeof(size));
  for (size_t i = 0; i < n_keys; i++) {
    hash_t key = keys[i];
    o.write((const char *)&key, sizeof(key));
    size_t n = offsets[i + 1] - offsets[i];
    o.write((const char *)&n, sizeof(n));
    o.write((const char *)&points[offsets[i]], n * sizeof(IntervalPoint));
  }
}

bool Sketch::loadIndexTSV(const std::string &path)
{  // winSketch.hpp:321-333
  std::ifstream in(path);
  if (!in) return false;
  std::string header;
  std::getline(in, header);
  long long seqId, strand, start, end;
  unsigned long long hash;
  while (in >> seqId >> strand >> start >> end >> hash)
    minmerIndex.push_back(make_mi(hash, (offset_t)start, (offset_t)end, (seqno_t)seqId, (strand_t)strand));
  return true;
}

/* PREFIX.index (winSketch.hpp:338-348): the header's record count n, then n records, read by `threads` threads in disjoint
 * ranges into alloc(n). A file too short for its header's count stops the run (exit status 1) with a message naming the
 * file and its size, before anything is allocated; bytes after the records are ignored, as in the reference. false: the
 * file cannot be opened. */
template <class Alloc>
static bool readIndexBinary(const std::string &path, int threads, Alloc &&alloc, uint64_t &n)
{
  const int fd = open(path.c_str(), O_RDONLY);
  if (fd < 0) return false;
  auto die = [&](const std::string &m) {
    std::cerr << "[mashmap-b200::skch::Sketch::build] ERROR: " << path << ": " << m << std::endl;
    exit(1);
  };
  struct stat sb;
  if (fstat(fd, &sb) != 0) die("cannot read its size");
  const uint64_t bytes = (uint64_t)sb.st_size;
  uint64_t count = 0;
  if (bytes < 8 || pread(fd, &count, 8, 0) != 8)
    die("the file holds " + std::to_string(bytes) + " bytes, too few for the 8-byte record count");
  if (count > (bytes - 8) / sizeof(MinmerInfo))
    die("the file holds " + std::to_string(bytes) + " bytes, too few for the " + std::to_string(count) +
        " records its header counts (8 + 24 x " + std::to_string(count) + " bytes)");
  char *dst = (char *)alloc(count);
  const uint64_t total = count * sizeof(MinmerInfo);
  const uint64_t T = (uint64_t)std::max(1, std::min(threads, 64));
  const uint64_t part = (total + T - 1) / T;
  std::atomic<bool> failed{false};
  std::vector<std::thread> pool;
  for (uint64_t t = 0; t < T; t++)
    pool.emplace_back([&, t]() {
      for (uint64_t at = std::min(total, t * part), end = std::min(total, at + part); at < end;) {
        const ssize_t got = pread(fd, dst + at, (size_t)std::min<uint64_t>(end - at, 1ULL << 30), (off_t)(8 + at));
        if (got <= 0) { failed = true; return; }
        at += (uint64_t)got;
      }
    });
  for (auto &th : pool) th.join();
  close(fd);
  if (failed) die("read error");
  n = count;
  return true;
}

bool Sketch::loadIndexBinary(const std::string &prefix)
{  // winSketch.hpp:338-348 (the interval points are rebuilt from the minmers, which gives the same lists)
  uint64_t n = 0;
  return readIndexBinary(prefix + ".index", param.threads, [&](uint64_t count) {
    minmerIndex.resize(count);
    return minmerIndex.data();
  }, n);
}

/* --loadIndex for the device: the records in pinned memory, as the file holds them (the device checks them); a TSV is
 * parsed into minmerIndex first and moved there */
bool Sketch::loadIndexForDevice()
{
  auto pinned = [&](uint64_t count) {
    void *p = nullptr;
    const uint64_t bytes = std::max<uint64_t>(count, 1) * sizeof(MinmerInfo);
    if (mm_host_alloc(&p, bytes) != MM_OK) {
      std::cerr << "[mashmap-b200::skch::Sketch::build] ERROR: cannot allocate " << bytes << " bytes of pinned host memory for the index" << std::endl;
      exit(1);
    }
    loaded_ = (MinmerInfo *)p;
    return loaded_;
  };
  const std::string path = param.loadIndexFilename.string();
  if (param.loadIndexFilename.extension() == ".tsv") {
    if (!loadIndexTSV(path)) return false;
    nLoaded_ = minmerIndex.size();
    if (nLoaded_) memcpy(pinned(nLoaded_), minmerIndex.data(), nLoaded_ * sizeof(MinmerInfo));
    else pinned(0);
    MI_Type().swap(minmerIndex);
    loadedFile_ = path;
    return true;
  }
  loadedFile_ = path + ".index";
  return readIndexBinary(loadedFile_, param.threads, pinned, nLoaded_);
}

}  // namespace skch
