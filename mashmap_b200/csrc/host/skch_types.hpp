/*
 * skch_types.hpp -- host-side mirror of the reference's public types for the mapping path, so that code
 * written against skch::Parameters / skch::Sketch / skch::Map / skch::MappingResult keeps compiling
 * (reference: src/map/include/base_types.hpp, map_parameters.hpp).
 * Only the members the path reads are kept; layouts of the records that cross the C ABI are the
 * ABI's (include/mashmap_b200.h), which are bit-compatible with the reference structs.
 */
#ifndef SKCH_TYPES_HPP
#define SKCH_TYPES_HPP

#include <cstdint>
#include <filesystem>
#include <functional>
#include <limits>
#include <string>
#include <vector>

#include "../../../include/mashmap_b200.h"

namespace skch {

typedef uint64_t hash_t;   // base_types.hpp:17
typedef int32_t offset_t;  // base_types.hpp:21 (LARGE_CONTIG is not supported: contigs < 2^31 bp)
typedef int32_t seqno_t;   // base_types.hpp:23
typedef int16_t strand_t;  // base_types.hpp:24
typedef int8_t side_t;     // base_types.hpp:25

typedef mm_minmer MinmerInfo;      // base_types.hpp:31-63 (same layout)
typedef mm_ipoint IntervalPoint;   // base_types.hpp:66-79 (same layout)

struct ContigInfo {  // base_types.hpp:96-100
  std::string name;
  offset_t len;
};

enum strnd : strand_t { FWD = 1, AMBIG = 0, REV = -1 };       // base_types.hpp:103-108
enum event : int { BEGIN = 1, END = 2 };                      // base_types.hpp:110-114
enum filter : int { MAP = 1, ONETOONE = 2, NONE = 3 };        // base_types.hpp:117-122
enum side : side_t { OPEN = 1, CLOSE = -1 };                  // base_types.hpp:125-129

// base_types.hpp:154-206. Same members and meaning; kmerComplexity is a long double in the reference,
// every value it ever holds is a float or a mean of floats computed in double.
struct MappingResult {
  offset_t queryLen;
  offset_t refStartPos;
  offset_t refEndPos;
  offset_t queryStartPos;
  offset_t queryEndPos;
  seqno_t refSeqId;
  seqno_t querySeqId;
  int blockLength;
  float nucIdentity;
  float nucIdentityUpperBound;
  int sketchSize;
  int conservedSketches;
  strand_t strand;
  int approxMatches;
  long double kmerComplexity;
  int n_merged;
  offset_t splitMappingId;
  uint8_t discard;
  bool selfMapFilter;

  offset_t qlen() { return queryEndPos - queryStartPos + 1; }
  offset_t rlen() { return refEndPos - refStartPos + 1; }
  size_t hash() const;  // base_types.hpp:188-204 (sparsifyMappings)
};
typedef std::vector<MappingResult> MappingResultsVector_t;

// map_parameters.hpp:32-80 (fields the path reads; same names)
struct Parameters {
  int kmerSize = 19;
  float kmer_pct_threshold = 0.001f;
  offset_t segLength = 5000;
  offset_t block_length = 5000;
  offset_t chain_gap = 5000;
  int alphabetSize = 4;
  offset_t referenceSize = 0;  // map_parameters.hpp:41: offset_t (int32): a file size >= 2 GiB wraps, and the wrapped value is
                               // sign-extended into recommendedSketchSize's uint64 parameter (parseCmdArgs.hpp:304,639) -- kept
  float percentageIdentity = 0.85f;
  bool stage2_full_scan = true;
  bool stage1_topANI_filter = true;
  float ANIDiff = 0.0f;
  float ANIDiffConf = 0.999f;
  int filterMode = filter::MAP;
  uint32_t numMappingsForSegment = 1;
  uint32_t numMappingsForShortSequence = 1;
  int threads = 1;
  std::vector<std::string> refSequences;
  std::vector<std::string> querySequences;
  std::string outFileName = "mashmap.out";
  std::filesystem::path saveIndexFilename;
  std::filesystem::path loadIndexFilename;
  bool split = true;
  bool lower_triangular = false;
  bool skip_self = false;
  bool skip_prefix = false;
  char prefix_delim = '\0';
  std::string target_list;
  std::string target_prefix;
  bool mergeMappings = true;
  bool keep_low_pct_id = true;
  bool report_ANI_percentage = false;
  bool filterLengthMismatches = false;
  float kmerComplexityThreshold = 0.0f;
  int sketchSize = 0;
  uint64_t sparsity_hash_threshold = std::numeric_limits<uint64_t>::max();
  bool legacy_output = false;
  // B200 additions (not in the reference)
  bool host_index = false;        // --hostIndex: build the reference index on the host (also for --saveIndex / --loadIndex)
  int device = 0;                 // CUDA device ordinal (--device)
  std::vector<int> devices;       // --devices 0-7 / 0,2,5: several GPUs driven by this process (empty = {device})
  int index_shards = 1;           // --indexShards N: the index cut by contig into N images, shard i on devices[i % D]
  uint64_t batch_bases = 1ULL << 30;  // query bases per device batch
  uint64_t sub_batch_bases = 640ULL << 20;  // a batch is mapped as sub-batches of this size on two pipelined lanes
  bool align = false;             // --align: NM:i / cg:Z tags from edlib NW over each printed mapping's region (on the device)
  // --alignMaxLen: longer query or target regions are printed without the tags. One warp aligns one mapping without a band:
  // 100 kb x 100 kb takes 1.9 s, 1 Mbp x 1 Mbp 341 s (H100 80GB HBM3, 400 W; scripts/map_align_perf.py)
  int64_t align_max_len = 100000;
  bool align_eqx = false;         // --eqx: cg:Z as an extended CIGAR (= / X / I / D)
  bool align_cs = false;          // --cs: also cs:Z, minimap2's short difference string
};

namespace fixed {  // map_parameters.hpp:86-102
constexpr double ss_table_max = 1000.0;
constexpr double pval_cutoff = 1e-3;
constexpr float confidence_interval = 0.95f;
constexpr float percentage_identity = 0.85f;
constexpr float ANIDiff = 0.0f;
constexpr float ANIDiffConf = 0.999f;
static const char *const VERSION = "3.1.3-b200";
}  // namespace fixed

}  // namespace skch

#endif
