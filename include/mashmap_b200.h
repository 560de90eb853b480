/*
 * mashmap_b200.h -- C ABI of the H100-native MashMap mapping hot path.
 *
 * The reference (marbl/MashMap v3.1.3) has no FFI/plugin boundary: its hot path is a set of
 * C++ member functions called once per query fragment from skch::Map::mapSingleQueryFrag
 * (src/map/include/computeMap.hpp:755-815). This header is the boundary a maintainer would bind
 * instead of those calls: plain pointers and sizes, int status codes, no C++/torch types, no
 * exceptions across the ABI. Each entry point cites the reference interface it replaces.
 * INTEGRATION.md shows the reference-side call sites (skch::Sketch / skch::Map) rewritten on top of it.
 *
 * All functions return MM_OK (0) or a negative MM_E* code; mm_last_error() gives the text.
 * There is NO CPU fallback: every compute entry point fails with MM_ENODEVICE when no sm_90
 * device is usable.
 */
#ifndef MASHMAP_B200_H
#define MASHMAP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MM_OK 0
#define MM_EINVAL (-1)     /* bad argument / unsupported parameter (e.g. k-mer size not compiled in)   */
#define MM_ENODEVICE (-2)  /* no CUDA device / wrong architecture: the product never computes on the CPU */
#define MM_ECUDA (-3)      /* a CUDA runtime call or kernel failed                                     */
#define MM_ENOMEM (-4)     /* device or host allocation failed                                         */
#define MM_ECAPACITY (-5)  /* caller-provided output capacity too small; *n_out holds the needed count  */
#define MM_ESTATE (-6)     /* call order violated (e.g. map before index upload)                       */

/* ---- record layouts (bit-compatible with the reference structs) ------------------------------- */

/* skch::MinmerInfo, base_types.hpp:31-63. 24 bytes. */
typedef struct mm_minmer {
  uint64_t hash;
  int32_t wpos;      /* query sketch: first position of the hash; reference index: first window  */
  int32_t wpos_end;  /* query sketch: last position;              reference index: one past last  */
  int32_t seqId;
  int16_t strand;    /* +1 FWD, 0 AMBIG, -1 REV (base_types.hpp:103-108) */
  int16_t _pad;
} mm_minmer;

/* skch::IntervalPoint, base_types.hpp:66-79. 24 bytes. */
typedef struct mm_ipoint {
  int32_t pos;
  int32_t _pad0;
  uint64_t hash;
  int32_t seqId;
  int8_t side;       /* +1 OPEN, -1 CLOSE (base_types.hpp:126-131) */
  int8_t _pad1[3];
} mm_ipoint;

/* skch::Map::L1_candidateLocus_t, computeMap.hpp:58-68, plus the owning segment. */
typedef struct mm_l1_candidate {
  int32_t seqId;
  int32_t rangeStartPos;
  int32_t rangeEndPos;
  int32_t intersectionSize;
  uint32_t segment;     /* index into the batch's segment table */
  uint32_t first_locus; /* index of this candidate's first mm_l2_locus */
  uint32_t n_loci;
  uint32_t _pad;
} mm_l1_candidate;

/* skch::Map::L2_mapLocus_t, computeMap.hpp:76-84. */
typedef struct mm_l2_locus {
  int32_t seqId;
  int32_t meanOptimalPos;
  int32_t optimalStart;
  int32_t optimalEnd;
  int32_t sharedSketchSize;
  int32_t strand;
} mm_l2_locus;

/* Per-segment result of getSeedHits (computeMap.hpp:817-843) + where its candidates are. */
typedef struct mm_segment_result {
  uint64_t sketch_max_hash;   /* Q.minmerTableQuery.back().hash BEFORE frequent-seed removal (:830) */
  int32_t sketch_raw_count;   /* Q.minmerTableQuery.size() before frequent-seed removal (:831)      */
  int32_t sketch_size;        /* Q.sketchSize after frequent-seed removal (:839)                    */
  int32_t n_points;           /* interval points gathered by getSeedIntervalPoints (:856-912)       */
  int32_t minimum_hits;       /* after the hypergeometric raise (:992-997); 0 if L1 returned early  */
  int32_t best_intersection;  /* bestIntersectionSize of sweep #1 (:982), uncapped                  */
  uint32_t first_candidate;   /* index of the first mm_l1_candidate of this segment                 */
  uint32_t n_candidates;      /* candidates in reference order (computeMap.hpp:1102-1115)           */
  uint32_t _pad;
} mm_segment_result;

/* The skch::Parameters fields the device path reads (map_parameters.hpp:32-80). */
typedef struct mm_params {
  int32_t kmer_size;            /* Parameters::kmerSize   */
  int32_t seg_length;           /* Parameters::segLength  */
  int32_t sketch_size;          /* Parameters::sketchSize */
  int32_t stage1_topani_filter; /* Parameters::stage1_topANI_filter (hypergeometric L1 filter)      */
  int32_t skip_self;            /* Parameters::skip_self        (computeMap.hpp:891)                */
  int32_t skip_prefix;          /* Parameters::skip_prefix      (computeMap.hpp:892)                */
  int32_t lower_triangular;     /* Parameters::lower_triangular (computeMap.hpp:893)                */
  int32_t _reserved[9];
} mm_params;

/* One query fragment = one call of mapSingleQueryFrag in the reference (computeMap.hpp:587-671). A fragment is normally at
 * most seg_length long; a longer one is a whole query mapped unsplit (--noSplit, :587-607) with windowLen = length -
 * seg_length (:933, :1306), up to length - kmer_size + 1 < 2^30 k-mer positions (the reference computes
 * (length - k + 1) * 2 in an int, :831). Results of such a fragment have the same layout (sketch_size slots, candidates,
 * loci); MM_DIAG_LONG_FRAGMENTS counts them. */
typedef struct mm_segment {
  uint64_t offset;      /* byte offset of the fragment in the batch's base buffer                  */
  int32_t length;       /* Q.len, kmer_size <= length (<= seg_length unless the query is unsplit)  */
  int32_t seq_counter;  /* Q.seqCounter (query sequence number; lower_triangular, :893)            */
  int32_t name_id;      /* id of the reference contig NAME equal to Q.seqName, or -1 (skip_self)   */
  int32_t ref_group;    /* Q.refGroup (getRefGroup, computeMap.hpp:164-177), or -1                 */
} mm_segment;

typedef struct mm_ctx mm_ctx;

/* ---- lifetime ---------------------------------------------------------------------------------- */

/* Replaces nothing in the reference (it has no device); one context per GPU / per process rank. */
/* Are these parameters inside the limits of the device path (k in 8..32; every mapping kernel launchable: one segment's
 * nibbles, twice, plus the sketch kernel's selection tables, and the L1 / L2 kernels' per-sketch state, each within 227 KB
 * of shared memory)? Needs no device: a caller checks BEFORE it reads and indexes a reference. MM_OK, or MM_EINVAL with
 * mm_last_error(NULL) naming the kernel that does not fit and the largest sketch size accepted for the segment length. */
int mm_params_check(const mm_params *params);
int mm_ctx_create(int device, const mm_params *params, mm_ctx **out);
int mm_ctx_destroy(mm_ctx *ctx);
const char *mm_last_error(const mm_ctx *ctx); /* ctx may be NULL: error of the last failed create */
int mm_ctx_device(const mm_ctx *ctx); /* the CUDA device the context lives on (-1 for NULL) */
/* Number of CUDA kernels this context has launched so far (bench.py's gpu_launches). */
uint64_t mm_kernel_launches(const mm_ctx *ctx);

/* Cumulative counts of the rare paths this context has taken (test / diagnostics only; nothing in the reference):
 * out[MM_DIAG_*]. */
#define MM_DIAG_L1_CTA_SEGMENTS 0  /* segments with more interval points than the warp path holds (CTA path)        */
#define MM_DIAG_L1_POOL_REGROW 1   /* L1 re-runs because the bump-allocated point pool was exhausted                  */
#define MM_DIAG_CAND_REGROW 2      /* re-runs because the candidate buffer was too small                              */
#define MM_DIAG_L2_GENERAL_CANDS 3 /* candidates redone by the general L2 kernel (more loci than the fixed slots / counter range) */
#define MM_DIAG_L2_LOCI_REGROW 4   /* L2 re-runs because the locus buffer was too small                               */
#define MM_DIAG_SKETCH_GENERAL_SEGMENTS 5 /* segments the fast sketch kernel handed to the general one (repeats, N-rich ...) */
#define MM_DIAG_LONG_FRAGMENTS 6   /* fragments longer than seg_length (windowLen > 0) sketched / mapped               */
int mm_ctx_diag(const mm_ctx *ctx, uint64_t out[8]);

/* ---- reference index -> device (replaces the in-memory members of skch::Sketch) ---------------- */

/* minmerIndex (winSketch.hpp:102, after dropFreqSeedSet :497-504), sorted by (seqId, wpos) as the
 * reference leaves it; minmerPosLookupIndex (winSketch.hpp:100-101) flattened as
 * keys[n_keys], offsets[n_keys+1], points[offsets[n_keys]] in reference per-key order;
 * key_is_freq[n_keys] = Sketch::isFreqSeed(key) (winSketch.hpp:506-509);
 * contig_len / contig_name_id / contig_group = Sketch::metadata[i].len, an id per distinct contig
 * name, and Map::refIdGroup[i] (computeMap.hpp:144-161). */
int mm_index_upload(mm_ctx *ctx,
                    const mm_minmer *minmer_index, uint64_t n_minmers,
                    const uint64_t *keys, const uint64_t *offsets, uint64_t n_keys,
                    const mm_ipoint *points, uint64_t n_points,
                    const uint8_t *key_is_freq,
                    const int32_t *contig_len, const int32_t *contig_name_id,
                    const int32_t *contig_group, int32_t n_contigs);

/* The same index BUILT ON THE DEVICE from the reference sequence: replaces the work of skch::Sketch's constructor --
 * build() / CommonFunc::addMinmers for every contig (winSketch.hpp:147-254, commonFunc.hpp:301-570), index() (:379-404),
 * computeFreqHist / computeFreqSeedSet / dropFreqSeedSet (:410-453, :488-504) -- and leaves the context as
 * mm_index_upload would (threshold tables still come from mm_tables_upload). seqs: the contigs as text, back to back
 * (contig i = [contig_offsets[i], contig_offsets[i+1])), in host memory or (seqs_on_device != 0) in device memory.
 * Lower case and IUPAC codes are normalised as the reference does. Records are the reference's; where its std::sort on
 * (wpos, wpos_end) leaves exact ties in an unspecified order, this builder keeps emission order (DESIGN.md).
 * keep_lookup != 0 keeps the flat lookup arrays on the device for mm_index_download. */
typedef struct mm_index_stats {
  uint64_t n_minmers;                /* minmerIndex.size() after dropFreqSeedSet                     */
  uint64_t n_minmers_before_filter;  /* "minmer windows picked from reference" (winSketch.hpp:228)  */
  uint64_t n_keys;                   /* "unique minmers" (:403)                                      */
  uint64_t n_points;                 /* interval points of all keys                                  */
  int32_t freq_threshold;            /* Sketch::getFreqThreshold(); INT32_MAX = consider all         */
  uint32_t n_chunks, n_fixed_chunks, fix_rounds; /* window scan: chunks, chunks re-scanned exactly, rounds */
  uint32_t hist_min_count, hist_max_count;       /* frequency histogram end points (:418-420)   */
  uint64_t hist_min_keys, hist_max_keys;
  float ms_scan, ms_post, ms_lookup, ms_total;
} mm_index_stats;
int mm_index_build(mm_ctx *ctx, const char *seqs, int seqs_on_device, const uint64_t *contig_offsets, int32_t n_contigs,
                   const int32_t *contig_name_id, const int32_t *contig_group, float kmer_pct_threshold, int keep_lookup,
                   mm_index_stats *stats);
/* Host copies of the index mm_index_build left on the device, in mm_index_upload's argument formats (any pointer may be
 * NULL; the lookup arrays need keep_lookup). Sizes: mm_index_stats. */
int mm_index_download(mm_ctx *ctx, mm_minmer *minmer_index, uint64_t *keys, uint64_t *offsets, mm_ipoint *points,
                      uint8_t *key_is_freq);

/* sketchCutoffs (Map::setProbs, computeMap.hpp:178-258) and
 * min_hits[s] = Stat::estimateMinimumHitsRelaxed(s, k, pi, 0.95) for s in [0, n_min_hits)
 * (map_stats.hpp:144-169; the reference recomputes it per fragment, computeMap.hpp:1144). */
int mm_tables_upload(mm_ctx *ctx, const int32_t *sketch_cutoffs, int32_t n_cutoffs,
                     const int32_t *min_hits, int32_t n_min_hits);

/* Multi-GPU: raw device images of everything mm_index_upload/mm_tables_upload put on the device,
 * so one rank can build and the others receive it with a single broadcast over NVLink
 * (SURVEY 8(e)). `blob` is a DEVICE pointer owned by the context; mm_index_adopt_blob takes a
 * device buffer filled by the broadcast and copies/adopts it. */
int mm_index_blob(mm_ctx *ctx, void **blob, uint64_t *n_bytes);
int mm_index_blob_alloc(mm_ctx *ctx, uint64_t n_bytes, void **blob);
int mm_index_adopt_blob(mm_ctx *ctx);
/* A second context on the SAME device that reads the index image of `src` (not copied, not owned): lets a host
 * pipeline keep several batches in flight (copies of one overlapping the kernels of another). `src` must outlive it;
 * if `src` later gets a new image (another upload, an adopted blob, new tables) this context follows it. */
int mm_ctx_share_index(mm_ctx *ctx, const mm_ctx *src);

/* ---- the hot path ------------------------------------------------------------------------------ */

/* K1 only: CommonFunc::sketchSequence (commonFunc.hpp:182-288) for every segment.
 * out_sketch[seg*sketch_size + j] for j < out_count[seg], ascending by hash; seqId = seq_counter.
 * A segment may be longer than seg_length (see mm_segment): it is sketched in pieces and merged on the device, with the
 * same result. Host buffers in, host buffers out. */
int mm_sketch_segments(mm_ctx *ctx, const char *bases, uint64_t n_bases,
                       const mm_segment *segments, uint64_t n_segments,
                       mm_minmer *out_sketch, int32_t *out_count);

/* mapSingleQueryFrag up to and including computeL2MappedRegions for every L1 candidate
 * (computeMap.hpp:755-815 -> :1129-1166 -> :1275-1451). Host buffers in/out; copies are inside.
 * The identity/threshold test and the HG early break (doL2Mapping, :1181-1267) are applied by the
 * caller on the returned records (they need only these integers; see INTEGRATION.md).
 * seg_results[n_segments]; candidates[cand_cap]; loci[loci_cap]. On MM_ECAPACITY n_candidates /
 * n_loci hold the required capacities and nothing else is valid. */
int mm_map_segments(mm_ctx *ctx, const char *bases, uint64_t n_bases,
                    const mm_segment *segments, uint64_t n_segments,
                    mm_segment_result *seg_results,
                    mm_l1_candidate *candidates, uint64_t cand_cap, uint64_t *n_candidates,
                    mm_l2_locus *loci, uint64_t loci_cap, uint64_t *n_loci);

/* The same with the bases already in the device's own input format, ONE NIBBLE PER BASE: base i of the batch is
 * (nibbles[i / 2] >> (4 * (i & 1))) & 15 = 2-bit code (A 0, C 1, T 2, G 3 = bits 1-2 of the upper-cased letter) | 8 for
 * every byte that is not ACGT after upper-casing -- makeUpperCaseAndValidDNA (commonFunc.hpp:75-107) folded into the
 * encoding. A host that touches every base anyway while it parses (skch::BatchMapper does) halves the PCIe traffic this
 * way; mm_map_segments does the same conversion on the device (kernel k_pack_bases). segments[i].offset counts BASES.
 * n_bases bases = (n_bases + 1) / 2 bytes. */
int mm_map_segments_packed(mm_ctx *ctx, const uint8_t *nibbles, uint64_t n_bases,
                           const mm_segment *segments, uint64_t n_segments,
                           mm_segment_result *seg_results,
                           mm_l1_candidate *candidates, uint64_t cand_cap, uint64_t *n_candidates,
                           mm_l2_locus *loci, uint64_t loci_cap, uint64_t *n_loci);

/* Same computation with the batch already resident in HBM (bench.py `value`):
 * upload once, run many times, fetch once. */
int mm_batch_upload(mm_ctx *ctx, const char *bases, uint64_t n_bases,
                    const mm_segment *segments, uint64_t n_segments);
int mm_batch_upload_packed(mm_ctx *ctx, const uint8_t *nibbles, uint64_t n_bases,
                           const mm_segment *segments, uint64_t n_segments);
int mm_map_resident(mm_ctx *ctx, uint64_t *n_candidates, uint64_t *n_loci);
int mm_batch_fetch(mm_ctx *ctx, mm_segment_result *seg_results,
                   mm_l1_candidate *candidates, uint64_t cand_cap,
                   mm_l2_locus *loci, uint64_t loci_cap);
/* Device sketches of the resident batch (after frequent-seed removal), for stage-level tests. */
int mm_batch_fetch_sketch(mm_ctx *ctx, mm_minmer *out_sketch, int32_t *out_count);

/* Scheduling hook for host pipelines that keep several contexts in flight on one device. The library calls
 * hook(user, phase, 1) before and hook(user, phase, 0) after
 *   MM_PHASE_UPLOAD_CHUNK  each <= 16 MiB piece of a batch upload (mm_batch_upload / mm_map_segments), and
 *   MM_PHASE_L2            the L2 record-preparation kernel of mm_map_resident / mm_map_segments (bandwidth-bound:
 *                          measured 4x slower while another context's PCIe upload is writing HBM, DESIGN.md section 5),
 * from the calling thread. A pipeline uses it to keep the two from overlapping (skch::BatchMapper does). NULL clears. */
#define MM_PHASE_UPLOAD_CHUNK 1
#define MM_PHASE_L2 2
typedef void (*mm_phase_hook)(void *user, int phase, int begin);
int mm_ctx_set_phase_hook(mm_ctx *ctx, mm_phase_hook hook, void *user);

/* How the calling thread waits for the device inside the library. 0 (default): it spins (cudaStreamSynchronize, lowest
 * latency: right when the host has a CPU to spare per context). 1: it sleeps on a blocking event, which costs tens of
 * microseconds per wait and frees the CPU: right when several contexts / processes share few host CPUs (one process per
 * GPU on a host whose CPUs are outnumbered, skch::BatchMapper switches by itself). Nothing in the reference to replace. */
int mm_ctx_set_wait_mode(mm_ctx *ctx, int blocking);

/* CUDA-event time in milliseconds of each stage of the last mm_map_resident / mm_map_segments:
 * [0] sketch kernel  [1] L1 kernel  [2] L2 kernel  [3] H2D  [4] D2H
 * [5] first kernel launch -> last kernel end (events on the launching stream; includes the two counter
 *     read-backs between kernels)  [6] L2 record-preparation kernel  [7] L2 scan kernel(s). */
int mm_last_stage_ms(const mm_ctx *ctx, float ms[8]);
/* ... and of the base-packing kernel that runs in front of the sketch kernel when the batch came in as text (0 for a
 * batch uploaded as nibbles). It is inside [5], not inside [0]. */
int mm_last_pack_ms(const mm_ctx *ctx, float *ms);

/* Pinned host memory for the caller's batch buffers (so the copies inside mm_map_segments run at full
 * PCIe rate). Plain malloc'ed buffers work too, only slower. */
int mm_host_alloc(void **ptr, uint64_t bytes);
int mm_host_free(void *ptr);

#ifdef __cplusplus
}
#endif
#endif /* MASHMAP_B200_H */
