/*
 * skch_map.hpp -- skch::Map: maps the query sequences on the device-resident reference index.
 *
 * Same constructor contract as the reference class (reference src/map/include/computeMap.hpp:53-139):
 * constructing it runs the whole mapping and writes param.outFileName; the optional callback is invoked
 * once per reported mapping, in output order, from the constructing thread (:100, :1802-1803).
 *
 * What moved to the GPU: everything mapSingleQueryFrag does per fragment up to the L2 loci
 * (computeMap.hpp:755-815 -> mm_map_segments of the C ABI). What stays on the host, restated (skch_tail.hpp):
 *   the identity / confidence-bound test and HG early break of doL2Mapping       (:1181-1267)
 *   read segmentation and query-coordinate rewriting of mapModule                (:587-672)
 *   mergeMappingsInRange, filterWeakMappings, filterByGroup + plane sweeps,
 *   filterFalseHighIdentity, mappingBoundarySanityCheck, sparsifyMappings        (:423-561, :1579-1750)
 *   reportReadMappings (PAF text)                                                (:1758-1805)
 *
 * skch::BatchMapper is the same machinery for reads that are already in memory: a batch of reads is laid out
 * in one (pinned) base buffer, fragmented with the reference's rule and mapped in parts of sub_batch_bases through a
 * three-stage pipeline (PCIe upload | kernels | record fetch + per-read host tail on param.threads threads), each part
 * on one of three device contexts that share the index image. skch::Map = FASTA reader + BatchMapper; output
 * order == input order, as in the reference (ThreadPool.hpp:187-211).
 */
#ifndef SKCH_MAP_HPP
#define SKCH_MAP_HPP

#include <functional>
#include <atomic>
#include <iostream>
#include <string>
#include <unordered_map>
#include <vector>

#include "skch_align.hpp"
#include "skch_index.hpp"
#include "skch_tail.hpp"
#include "skch_types.hpp"

struct mm_ctx;

namespace skch {

/* one device batch of reads */
struct ReadBatch {
  /* pinned host memory (BatchMapper::allocBases) holding the reads in the device's input format: ONE NIBBLE PER BASE
   * (seqio::pack_bases; base i of the batch in byte i / 2). capacity / used count BASES; every read starts at a multiple
   * of READ_ALIGN bases, so two threads packing neighbouring reads never share a byte (or a cache line's word). */
  static constexpr uint64_t READ_ALIGN = 32;
  char *bases = nullptr;
  uint64_t capacity = 0, used = 0;
  uint8_t *nibbles(uint64_t base_offset) const { return (uint8_t *)bases + (base_offset >> 1); }
  std::vector<mm_segment> segs;
  std::vector<ReadRec> reads;
  void clear() { used = 0; segs.clear(); reads.clear(); }
};

class BatchMapper {
 public:
  BatchMapper(const Parameters &p, const Sketch &refsketch);  // creates the device context, uploads index + tables
  ~BatchMapper();
  BatchMapper(const BatchMapper &) = delete;

  char *allocBases(uint64_t n_bases);  // room for n_bases bases (n_bases / 2 bytes + slack)
  void freeBases(char *p);
  /* mapModule's fragmenting (computeMap.hpp:587-671): appends the read's fragments to the batch.
   * `seq` (text) is packed into the batch; nullptr = the caller packs the bases itself at b.nibbles(offset of the read's
   * first fragment) (the bulk FASTA path does that from all host threads). */
  void addRead(ReadBatch &b, const std::string &name, const char *seq, offset_t len, seqno_t seqCounter) const;
  /* one device call + the host tail; results[r] = final mappings of batch.reads[r]; text[r] = their PAF lines */
  void mapBatch(const ReadBatch &b, std::vector<MappingResultsVector_t> &results, std::vector<std::string> *text,
                const std::vector<ContigInfo> *qmetadata);

  /* -f one-to-one, the run-wide step of mapQuery (computeMap.hpp:358-405): all mappings of all reads go through the
   * reference-axis plane sweep together (per query prefix group with -Y), are sorted by (query id, query start, ref id,
   * ref start) and formatted. Works on whatever set the caller hands over -- the mappings of one process, or the
   * records gathered from all ranks (MappingResult is a POD, base_types.hpp:152-153). */
  void finalizeOneToOne(MappingResultsVector_t &allReadMappings, const std::vector<ContigInfo> &qmetadata, std::string &paf) const;
  /* --align after finalizeOneToOne: appends NM:i / cg:Z to the lines of paf, which are maps in order; query(id) = the
   * nibbles of query id. The mappings are split into one contiguous slice per device. (Outside one-to-one mode mapBatch
   * aligns each part after its host tail.) */
  void alignOneToOne(const MappingResultsVector_t &maps, const std::function<const uint8_t *(seqno_t)> &query, std::string &paf);
  void reportAlignment() const;  // --align: totals of the run to stderr

  /* --indexShards: cuts contigs [0, len.size()) into n_shards contiguous ranges balanced by bases; with byGroup (-Y) a cut
   * only falls where group[] changes, so that no prefix group spans two shards. first[i] = first contig of shard i
   * (first[n_shards] = the number of contigs). Returns "" or why the reference cannot be cut so. */
  static std::string planShards(const std::vector<uint64_t> &len, const std::vector<int> &group, bool byGroup, int n_shards,
                                std::vector<int32_t> &first);
  int getRefGroup(const std::string &seqName) const;  // computeMap.hpp:164-177
  const std::vector<int> &refGroups() const { return refIdGroup; }
  const MapTail &tail() const { return *tail_; }
  mm_ctx *context() const { return ctx; }
  int deviceCount() const { return (int)groups.size(); }
  double secondsDevice = 0, secondsHostTail = 0;
  // totals of the last mapBatch, accumulated by the tail workers: text bytes, reads with a mapping, mappings
  std::atomic<uint64_t> lastTextBytes{0}, lastMappedReads{0}, lastMappings{0};
  float lastStageMs[8] = {0};

 private:
  const Parameters &param;
  const Sketch &refSketch;
  std::vector<int> sketchCutoffs;  // computeMap.hpp:109
  std::vector<int> refIdGroup;     // computeMap.hpp:113
  std::vector<int> minHits;        // estimateMinimumHitsRelaxed by Q.sketchSize (computeMap.hpp:1144)
  std::unordered_map<std::string, int> refNameId;
  std::vector<int> contigNameId;
  mm_ctx *ctx = nullptr;   // the first device's context: owns the index image that was uploaded
  MapTail *tail_ = nullptr;
  class WorkerPool;
  struct Lane {  // per pipeline lane: device context (own stream + buffers) and its host-side record buffers
    mm_ctx *ctx = nullptr;
    std::vector<mm_segment> segs;
    /* the records mm_batch_fetch copies back live in pinned memory: a device->host copy into pageable memory goes through
     * the driver's staging buffer at ~8 GB/s and costs host CPU time on top (1.8 ms per 134 k-fragment part) */
    template <class T>
    struct PinnedArray {
      T *p = nullptr;
      size_t cap = 0;
      T *data() const { return p; }
      size_t size() const { return cap; }
      void reserve(size_t n)
      {
        if (n <= cap) return;
        if (p) mm_host_free(p);
        p = nullptr; cap = 0;
        void *q = nullptr;
        if (mm_host_alloc(&q, n * sizeof(T)) != MM_OK) { std::cerr << "[mashmap-b200] ERROR: cannot pin " << n * sizeof(T) << " bytes" << std::endl; exit(1); }
        p = (T *)q; cap = n;
      }
      void release() { if (p) mm_host_free(p); p = nullptr; cap = 0; }
    };
    PinnedArray<mm_segment_result> segRes;
    PinnedArray<mm_l1_candidate> cands;
    PinnedArray<mm_l2_locus> loci;
    size_t r0 = 0, r1 = 0, s0 = 0, nseg = 0;  // the part in flight on this lane
    uint64_t nc = 0, nl = 0;
    double secDevice = 0, secTail = 0, msUpload = 0, msCompute = 0;
    float stageMs[8] = {0};
  };
  // scheduler state of the phase hook: batch uploads wait while the L2 kernels of another lane run
  struct Gate;
  static void phaseHook(void *user, int phase, int begin);
  static constexpr int MAX_LANES = 3;
  /* One group per GPU this process drives (--devices): its own index image (replicated from the first device with one
   * grouped NCCL broadcast, mm_index_replicate), its own three pipeline lanes and gate, its own share of the host-tail
   * threads. The parts of a batch are dealt to the groups round robin (a read lives in one part, so output order and
   * content do not depend on the number of devices). */
  struct DeviceGroup {
    int device = 0;
    mm_ctx *owner = nullptr;  // holds this device's index image
    Lane lanes[MAX_LANES];
    int nLanes = 1;
    Gate *gate = nullptr;
    WorkerPool *tailPool = nullptr;  // persistent threads of the per-read host tail
    MappingAligner *aligner = nullptr;  // --align; used by the thread that finishes this device's parts
    bool blockingWaits = false;  // host waits sleep on events instead of spinning (few CPUs per device)
    int tailThreads = 1;
  };
  std::vector<DeviceGroup *> groups;
  /* --indexShards N > 1: shard i (contigs [shardFirst[i], shardFirst[i + 1])) is the index image of shards[i].ctx, on
   * devices[i % D]; every part of a batch runs on all of them (one lane) and their records are merged per segment */
  struct Shard {
    mm_ctx *ctx = nullptr;
    std::vector<mm_segment_result> segRes;
    std::vector<mm_l1_candidate> cands;
    std::vector<mm_l2_locus> loci;
    std::vector<int32_t> best;
    uint64_t nc = 0, nl = 0;
  };
  std::vector<Shard> shards;
  std::vector<int32_t> shardFirst;
  void buildShards(const mm_params &mp);
  void shardsCompute(Lane &ln);
  void shardsFetch(Lane &ln);
  void setRefGroups();
  void laneUpload(Lane &ln, const ReadBatch &b, size_t r0, size_t r1);
  void laneCompute(Lane &ln);
  void laneFinish(DeviceGroup &g, Lane &ln, const ReadBatch &b, std::vector<MappingResultsVector_t> &results,
                  std::vector<std::string> *text, const std::vector<ContigInfo> *qmetadata);
  void runGroup(DeviceGroup &g, const ReadBatch &b, const std::vector<std::pair<size_t, size_t>> &parts, size_t first, size_t step,
                std::vector<MappingResultsVector_t> &results, std::vector<std::string> *text, const std::vector<ContigInfo> *qmetadata);
};

class Map {
 public:
  struct L1_candidateLocus_t {  // computeMap.hpp:58-68
    seqno_t seqId;
    offset_t rangeStartPos;
    offset_t rangeEndPos;
    int intersectionSize;
  };
  struct L2_mapLocus_t {  // computeMap.hpp:76-84
    seqno_t seqId;
    offset_t meanOptimalPos;
    offset_t optimalStart;
    offset_t optimalEnd;
    int sharedSketchSize;
    strand_t strand;
  };
  typedef std::function<void(const MappingResult &)> PostProcessResultsFn_t;  // computeMap.hpp:100

  Map(const Parameters &p, const Sketch &refsketch, PostProcessResultsFn_t f = nullptr);  // :123-139
  ~Map();

  static void insertL2ResultsToVec(MappingResultsVector_t &v, const MappingResult &r) { v.push_back(r); }  // :1813

  // timing of the run (seconds), for the driver program
  double secondsDevice = 0, secondsHostTail = 0, secondsInput = 0;
  uint64_t totalQueryBases = 0;

 private:
  struct Impl;
  Impl *impl;
};

}  // namespace skch
#endif
