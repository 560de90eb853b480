/*
 * skch_index.hpp -- skch::Sketch: the reference minmer index (reference src/map/include/winSketch.hpp).
 *
 * Same constructor contract and public members as the reference class (winSketch.hpp:57-511): the
 * constructor builds and indexes (blocking); `metadata`, `minmerIndex`, the frequent-seed predicate and
 * threshold are public. The hash -> interval-point map (`minmerPosLookupIndex`, winSketch.hpp:100-101)
 * is kept flattened (keys ascending / offsets / points), which is the form the device consumes.
 *
 * Round-1 builder: minmer windows are computed on the host by a step-for-step restatement of
 * CommonFunc::addMinmers (commonFunc.hpp:301-570), one task per contig, because every record's wpos is an
 * L2 evaluation point and the reference's record boundaries (vote-sum zero crossings, chunking, the
 * unstable sort's tie order) are only reproducible by following the same steps with the same libstdc++
 * (SURVEY 7.2, A.6). A device builder is the first "next" row of SURVEY 8(f).
 */
#ifndef SKCH_INDEX_HPP
#define SKCH_INDEX_HPP

#include <limits>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "skch_types.hpp"

namespace skch {

template <class T>
struct default_init_allocator : std::allocator<T> {
  template <class U> struct rebind { typedef default_init_allocator<U> other; };
  default_init_allocator() = default;
  template <class U> default_init_allocator(const default_init_allocator<U> &) {}
  template <class U> void construct(U *p) noexcept(std::is_nothrow_default_constructible<U>::value) { ::new ((void *)p) U; }
  template <class U, class... A> void construct(U *p, A &&...a) { ::new ((void *)p) U(std::forward<A>(a)...); }
};
template <class T> using BigVec = std::vector<T, default_init_allocator<T>>;

namespace CommonFunc {
/* commonFunc.hpp:301-570 */
void addMinmers(std::vector<MinmerInfo> &minmerIndex, char *seq, offset_t len, int kmerSize, int windowSize,
                int alphabetSize, int sketchSize, seqno_t seqCounter, bool stable_ties = false);
/* the post-processing of addMinmers (commonFunc.hpp:522-568) over records in emission order */
void finishMinmers(std::vector<MinmerInfo> &out, int windowSize, bool stable_ties = false);
/* the chunked + stitched scan the GPU builder performs, on the host (tests): returns the number of re-scanned chunks */
int addMinmersChunked(std::vector<MinmerInfo> &out, char *seq, offset_t len, int kmerSize, int windowSize, int sketchSize,
                      seqno_t seqCounter, offset_t chunk, offset_t warm);
/* commonFunc.hpp:591-603 */
uint64_t getReferenceSize(const std::vector<std::string> &refSequences);
}  // namespace CommonFunc

/* computeFreqHist's threshold (winSketch.hpp:418-449) over the histogram {interval points -> keys} of totalUniqueMinmers
 * keys, with the reference's log lines; INT_MAX = consider all minmers */
int computeFreqThreshold(const std::map<int, int> &hist, int64_t totalUniqueMinmers, float kmer_pct_threshold);
/* The frequent seeds of a reference indexed in contig shards: keys[i][0, n[i]) are shard i's distinct hashes (ascending) and
 * counts[i] their interval points. The histogram is the one of the union (a hash counts the points of every shard; each
 * distinct hash is one key), so threshold, log lines and the returned hashes (ascending, count >= threshold) are those of
 * the unsharded index. */
std::vector<hash_t> globalFrequentSeeds(const std::vector<const hash_t *> &keys, const std::vector<const uint32_t *> &counts,
                                        const std::vector<uint64_t> &n, float kmer_pct_threshold, int &threshold, uint64_t &n_unique);

class Sketch {
 public:
  typedef std::vector<MinmerInfo> MI_Type;

  explicit Sketch(const Parameters &p);  // winSketch.hpp:122-138: build + index + frequency filter
  ~Sketch();
  // same pipeline on sequences already in memory (seqs[i] has metadata[i].len bases); used by bench.py
  Sketch(const Parameters &p, const std::vector<ContigInfo> &contigs, const std::vector<const char *> &seqs);
  // index + frequency filter over an existing minmer list (winSketch.hpp:379-504 without build())
  Sketch(const Parameters &p, const std::vector<ContigInfo> &contigs, MI_Type &&minmers);

  std::vector<ContigInfo> metadata;          // winSketch.hpp:79
  std::vector<int> sequencesByFileInfo;      // winSketch.hpp:88
  MI_Type minmerIndex;                       // winSketch.hpp:102 (after dropFreqSeedSet)

  // minmerPosLookupIndex (winSketch.hpp:101), flattened: keys ascending; points of keys[i] are
  // lookupPoints[lookupOffsets[i] .. lookupOffsets[i+1]) in reference per-key order
  // (BigVec: resize() leaves trivially-constructible elements uninitialised -- these arrays are filled by all threads
  //  right away, and zero-filling 12 GB of points on one thread first cost seconds at 3 Gbp)
  BigVec<hash_t> lookupKeys;
  BigVec<uint64_t> lookupOffsets;
  BigVec<IntervalPoint> lookupPoints;
  std::vector<uint8_t> lookupKeyIsFreq;      // frequentSeeds membership per key (winSketch.hpp:488-495)

  /* The index is built ON THE DEVICE unless --hostIndex is given (by skch::BatchMapper, which owns the device context):
   * the constructor then only reads the contigs, and with --loadIndex the file's records; minmerIndex and the lookup
   * arrays stay empty on the host. From the text (mm_index_build) or from the loaded records (mm_index_build_minmers);
   * with --saveIndex, after either, the build keeps what the files hold and saveDeviceIndex writes them. --hostIndex
   * keeps everything on the host, --saveIndex and --loadIndex included. */
  bool deviceBuildPending() const { return deviceText_ != nullptr; }
  const char *deviceText() const { return deviceText_; }
  const std::vector<uint64_t> &deviceTextOffsets() const { return deviceTextOffsets_; }
  bool deviceLoadPending() const { return loaded_ != nullptr; }
  const MinmerInfo *loadedRecords() const { return loaded_; }  // pinned host memory (mm_host_alloc)
  uint64_t loadedCount() const { return nLoaded_; }
  const std::string &loadedFile() const { return loadedFile_; }
  void deviceBuildDone(int freq_threshold) const;  // releases the text or the loaded records, records the threshold
  /* --saveIndex of an index mm_index_build or mm_index_build_minmers made with MM_KEEP_LOOKUP | MM_KEEP_UNFILTERED (st:
   * its statistics): downloads the records before the frequent-seed drop and the lookup, releases what the build kept on
   * the device, and writes the files finish() would write (records' _pad bytes zero) */
  void saveDeviceIndex(mm_ctx *ctx, const mm_index_stats &st) const;

  /* --align: the bases of contig i (metadata[i]) as nibbles (seqio::pack_bases: ACGT, everything else N), base 0 in the
   * low nibble of the first byte. Read with the contigs in every index mode and kept for the whole run (not kept by the
   * constructor that takes a minmer list). */
  const uint8_t *refNibbles(seqno_t i) const { return refNibbles_.data() + refNibbleOffsets_[(size_t)i]; }

  int getFreqThreshold() const { return freqThreshold; }   // winSketch.hpp:483-486
  bool isFreqSeed(hash_t h) const;                         // winSketch.hpp:506-509
  bool isMinmerIndexEnd(MI_Type::const_iterator it) const { return it == minmerIndex.end(); }
  MI_Type::const_iterator getMinmerIndexEnd() const { return minmerIndex.end(); }

  // --saveIndex / --loadIndex (winSketch.hpp:270-374): TSV and PREFIX.index/.map binary formats
  static void saveIndexTSV(const std::string &path, const MinmerInfo *mi, size_t n);
  static void saveIndexBinary(const std::string &prefix, const MinmerInfo *mi, size_t n);
  static void savePosListBinary(const std::string &prefix, const hash_t *keys, const uint64_t *offsets, const IntervalPoint *points,
                                size_t n_keys);

 private:
  const Parameters &param;
  mutable int freqThreshold = std::numeric_limits<int>::max();
  bool saving_ = false;
  mutable char *deviceText_ = nullptr;           // contigs back to back (text), until the device has built the index
  mutable std::vector<uint64_t> deviceTextOffsets_;
  mutable MinmerInfo *loaded_ = nullptr;         // --loadIndex: the file's records, until the device has indexed them
  uint64_t nLoaded_ = 0;
  std::string loadedFile_;
  BigVec<uint8_t> refNibbles_;                   // --align only
  std::vector<uint64_t> refNibbleOffsets_;       // byte offset of each contig in refNibbles_

  void build();
  void keepForAlign(const char *seq, size_t len);  // appends a contig to refNibbles_
  void buildFromMemory(const std::vector<const char *> &seqs);
  void finish();
  // the --saveIndex files (the records before the frequent-seed drop, and the lookup), as the extension asks
  void writeIndexFiles(const MinmerInfo *mi, size_t n, const hash_t *keys, const uint64_t *offsets, const IntervalPoint *points,
                       size_t n_keys) const;
  bool loadIndexForDevice();
  void index();
  void computeFreqHist();
  void dropFreqSeedSet();
  bool loadIndexTSV(const std::string &path);
  bool loadIndexBinary(const std::string &prefix);
};

}  // namespace skch
#endif
