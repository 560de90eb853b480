/*
 * skch_cview.cpp -- a flat C view of the host-side classes for the ctypes tests (no GPU needed):
 * the statistics tables, the host index builder, and the host tail fed with externally produced records.
 * Not part of the drop-in boundary (that is include/mashmap_b200.h + the skch:: classes).
 */
#include <algorithm>
#include <memory>
#include <atomic>
#include <chrono>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sstream>
#include <random>
#include <string>
#include <vector>

#include "skch_args.hpp"
#include "skch_index.hpp"
#include "skch_map.hpp"
#include "skch_seqio.hpp"
#include "skch_stats.hpp"
#include "skch_filter.hpp"
#include "skch_tail.hpp"
#include "../mm_inflate.h"

#include <zlib.h>

using namespace skch;

extern "C" {

double skch_binomial_Q(unsigned k, double p, unsigned n) { return Stat::binomial_Q(k, p, n); }
float skch_j2md(float j, int k) { return Stat::j2md(j, k); }
float skch_md2j(float d, int k) { return Stat::md2j(d, k); }
float skch_md_lower_bound(float d, int s, int k) { return Stat::md_lower_bound(d, s, k, fixed::confidence_interval); }
int skch_min_hits(int s, int k, float pi) { return Stat::estimateMinimumHitsRelaxed(s, k, pi, fixed::confidence_interval); }
int64_t skch_recommended_sketch_size(int k, float pi, int64_t segLength, uint64_t refSize)
{
  return Stat::recommendedSketchSize(fixed::pval_cutoff, fixed::confidence_interval, k, 4, pi, segLength, refSize);
}
/* gsl_ran_hypergeometric_pdf(k, n1, n2, t) for k = 0..t as the product computes it (tests/test_stats_scipy_cpu.py) */
int skch_hypergeometric_pmf_row(unsigned n1, unsigned n2, unsigned t, double *out, int cap)
{
  std::vector<double> row;
  Stat::hypergeometric_pmf_row(n1, n2, t, row);
  for (int i = 0; i < (int)row.size() && i < cap; i++) out[i] = row[(size_t)i];
  return (int)row.size();
}
int skch_sketch_cutoffs(int sketchSize, int k, float aniDiff, float aniDiffConf, int enabled, int *out, int cap)
{
  std::vector<int> c = Stat::sketchCutoffs(sketchSize, k, aniDiff, aniDiffConf, enabled != 0);
  for (int i = 0; i < (int)c.size() && i < cap; i++) out[i] = c[i];
  return (int)c.size();
}

int64_t skch_add_minmers_ex(const char *seq, int64_t len, int k, int w, int s, int seqId, mm_minmer *out, int64_t cap, int stable_ties);
int64_t skch_add_minmers(const char *seq, int64_t len, int k, int w, int s, int seqId, mm_minmer *out, int64_t cap)
{
  return skch_add_minmers_ex(seq, len, k, w, s, seqId, out, cap, 0);
}
/* stable_ties: records with equal (wpos, wpos_end) stay in emission order (the GPU builder's order) instead of std::sort's */
int64_t skch_add_minmers_ex(const char *seq, int64_t len, int k, int w, int s, int seqId, mm_minmer *out, int64_t cap, int stable_ties)
{
  std::string buf(seq, (size_t)len);
  std::vector<MinmerInfo> v;
  CommonFunc::addMinmers(v, &buf[0], (offset_t)len, k, w, 4, s, seqId, stable_ties != 0);
  if ((int64_t)v.size() > cap) return -(int64_t)v.size();
  if (!v.empty()) memcpy(out, v.data(), v.size() * sizeof(mm_minmer));
  return (int64_t)v.size();
}

/* ---- the reference index as flat arrays (keys ascending / offsets / points / frequent flags) ---- */
struct IndexHandle {
  Parameters p;
  Sketch *sk = nullptr;
};

/* index + frequency filter over an existing minmer list */
/* the chunked + stitched scan (what the GPU builder does per chunk) on the host; *rescans = chunks scanned from the previous
 * chunk's exact state instead of a warm-up */
int64_t skch_add_minmers_chunked(const char *seq, int64_t len, int k, int w, int s, int seqId, int64_t chunk, int64_t warm,
                                 mm_minmer *out, int64_t cap, int32_t *rescans)
{
  std::string buf(seq, (size_t)len);
  std::vector<MinmerInfo> v;
  const int r = CommonFunc::addMinmersChunked(v, &buf[0], (offset_t)len, k, w, s, seqId, (offset_t)chunk, (offset_t)warm);
  if (rescans) *rescans = r;
  for (size_t i = 0; i < v.size() && (int64_t)i < cap; i++) out[i] = v[i];
  return (int64_t)v.size();
}

void *skch_index_from_minmers(const mm_minmer *mi, uint64_t n, int n_contigs, float kmer_pct_threshold)
{
  IndexHandle *h = new IndexHandle();
  h->p.kmer_pct_threshold = kmer_pct_threshold;
  std::vector<ContigInfo> meta;
  for (int i = 0; i < n_contigs; i++) meta.push_back(ContigInfo{std::to_string(i), 0});
  Sketch::MI_Type v(mi, mi + n);
  h->sk = new Sketch(h->p, meta, std::move(v));
  return h;
}

/* full host build from sequences in memory: seqs = concatenated contigs, offs[n_contigs+1] */
void *skch_index_build(const char *seqs, const uint64_t *offs, int n_contigs, int k, int segLength, int sketchSize, int threads,
                       float kmer_pct_threshold)
{
  IndexHandle *h = new IndexHandle();
  h->p.kmerSize = k; h->p.segLength = segLength; h->p.sketchSize = sketchSize; h->p.threads = threads;
  h->p.kmer_pct_threshold = kmer_pct_threshold;
  std::vector<ContigInfo> meta;
  std::vector<const char *> ptrs;
  for (int i = 0; i < n_contigs; i++) {
    meta.push_back(ContigInfo{"ctg" + std::to_string(i), (offset_t)(offs[i + 1] - offs[i])});
    ptrs.push_back(seqs + offs[i]);
  }
  h->sk = new Sketch(h->p, meta, ptrs);
  return h;
}

/* skch::Sketch exactly as the driver program builds it: the reference's command line (reference
 * parseCmdArgs.hpp) -> Parameters -> Sketch(param), including --saveIndex / --loadIndex. No device needed. */
void *skch_index_from_cli(int argc, const char **argv)
{
  IndexHandle *h = new IndexHandle();
  std::vector<std::string> store;
  store.push_back("mashmap-b200");
  for (int i = 0; i < argc; i++) store.push_back(argv[i]);
  std::vector<char *> av;
  for (auto &x : store) av.push_back(&x[0]);
  parseandSave((int)av.size(), av.data(), h->p);
  h->p.host_index = true;  /* this view exposes the host arrays of the index: built on the host (the CLI builds it on the device) */
  h->sk = new Sketch(h->p);
  return h;
}
/* command line -> Parameters only (no Sketch): for option-parser tests that must not read the reference file */
void *skch_params_from_cli(int argc, const char **argv)
{
  IndexHandle *h = new IndexHandle();
  std::vector<std::string> store;
  store.push_back("mashmap-b200");
  for (int i = 0; i < argc; i++) store.push_back(argv[i]);
  std::vector<char *> av;
  for (auto &x : store) av.push_back(&x[0]);
  parseandSave((int)av.size(), av.data(), h->p);
  return h;
}
int skch_index_sketch_size(void *hv) { return ((IndexHandle *)hv)->p.sketchSize; }

/* the Parameters the command line produced, in the field order of the oracle's orc_params (tests/refh.py OrcParams) */
struct skch_params_view {
  int32_t kmerSize, segLength, sketchSize, alphabetSize;
  float percentageIdentity;
  int32_t filterMode, numMappingsForSegment, numMappingsForShortSequence, block_length, chain_gap, split, mergeMappings,
      stage1_topANI_filter;
  float ANIDiff, ANIDiffConf;
  int32_t stage2_full_scan, keep_low_pct_id;
  float kmer_pct_threshold, kmerComplexityThreshold;
  int32_t skip_self, skip_prefix, prefix_delim, lower_triangular, filterLengthMismatches, legacy_output, report_ANI_percentage;
  uint64_t sparsity_hash_threshold, referenceSize;
};
void skch_index_params(void *hv, skch_params_view *o)
{
  const Parameters &p = ((IndexHandle *)hv)->p;
  memset(o, 0, sizeof(*o));
  o->kmerSize = p.kmerSize; o->segLength = p.segLength; o->sketchSize = p.sketchSize; o->alphabetSize = p.alphabetSize;
  o->percentageIdentity = p.percentageIdentity; o->filterMode = p.filterMode;
  o->numMappingsForSegment = (int32_t)p.numMappingsForSegment; o->numMappingsForShortSequence = (int32_t)p.numMappingsForShortSequence;
  o->block_length = p.block_length; o->chain_gap = p.chain_gap; o->split = p.split; o->mergeMappings = p.mergeMappings;
  o->stage1_topANI_filter = p.stage1_topANI_filter; o->ANIDiff = p.ANIDiff; o->ANIDiffConf = p.ANIDiffConf;
  o->stage2_full_scan = p.stage2_full_scan; o->keep_low_pct_id = p.keep_low_pct_id; o->kmer_pct_threshold = p.kmer_pct_threshold;
  o->kmerComplexityThreshold = p.kmerComplexityThreshold; o->skip_self = p.skip_self; o->skip_prefix = p.skip_prefix;
  o->prefix_delim = p.prefix_delim; o->lower_triangular = p.lower_triangular; o->filterLengthMismatches = p.filterLengthMismatches;
  o->legacy_output = p.legacy_output; o->report_ANI_percentage = p.report_ANI_percentage;
  o->sparsity_hash_threshold = p.sparsity_hash_threshold; o->referenceSize = (uint64_t)p.referenceSize; /* sign-extends, as the reference's use does */
}

/* contig metadata only (ranks that receive the device index image by broadcast) */
void *skch_index_metadata_only(int n_contigs, int contig_len, int k, int segLength, int sketchSize)
{
  IndexHandle *h = new IndexHandle();
  h->p.kmerSize = k; h->p.segLength = segLength; h->p.sketchSize = sketchSize;
  std::vector<ContigInfo> meta;
  for (int i = 0; i < n_contigs; i++) meta.push_back(ContigInfo{"ctg" + std::to_string(i), (offset_t)contig_len});
  h->sk = new Sketch(h->p, meta, Sketch::MI_Type());
  return h;
}

void skch_index_destroy(void *hv)
{
  IndexHandle *h = (IndexHandle *)hv;
  if (h) { delete h->sk; delete h; }
}
void skch_index_sizes(void *hv, uint64_t *n_minmers, uint64_t *n_keys, uint64_t *n_points, int32_t *freq_threshold)
{
  Sketch *s = ((IndexHandle *)hv)->sk;
  if (!s) { *n_minmers = *n_keys = *n_points = 0; *freq_threshold = 0; return; } /* parameters-only handle */
  *n_minmers = s->minmerIndex.size(); *n_keys = s->lookupKeys.size(); *n_points = s->lookupPoints.size();
  *freq_threshold = s->getFreqThreshold();
}
void skch_index_copy(void *hv, mm_minmer *mi, uint64_t *keys, uint64_t *offs, mm_ipoint *pts, uint8_t *is_freq)
{
  Sketch *s = ((IndexHandle *)hv)->sk;
  if (mi && !s->minmerIndex.empty()) memcpy(mi, s->minmerIndex.data(), s->minmerIndex.size() * sizeof(mm_minmer));
  if (keys && !s->lookupKeys.empty()) memcpy(keys, s->lookupKeys.data(), s->lookupKeys.size() * 8);
  if (offs) memcpy(offs, s->lookupOffsets.data(), s->lookupOffsets.size() * 8);
  if (pts && !s->lookupPoints.empty()) memcpy(pts, s->lookupPoints.data(), s->lookupPoints.size() * sizeof(mm_ipoint));
  if (is_freq && !s->lookupKeyIsFreq.empty()) memcpy(is_freq, s->lookupKeyIsFreq.data(), s->lookupKeyIsFreq.size());
}
/* upload straight into a device context (no copies through Python) */
int skch_index_upload(void *hv, mm_ctx *ctx)
{
  Sketch *s = ((IndexHandle *)hv)->sk;
  std::vector<int32_t> clen(s->metadata.size());
  for (size_t i = 0; i < clen.size(); i++) clen[i] = s->metadata[i].len;
  return mm_index_upload(ctx, s->minmerIndex.data(), s->minmerIndex.size(), s->lookupKeys.data(), s->lookupOffsets.data(),
                         s->lookupKeys.size(), s->lookupPoints.data(), s->lookupPoints.size(), s->lookupKeyIsFreq.data(),
                         clen.data(), nullptr, nullptr, (int32_t)clen.size());
}

/* ---- BatchMapper on reads already in (pinned) memory: the end-to-end call bench.py times ---- */
struct BmHandle {
  IndexHandle *ih;
  BatchMapper *bm;
  std::vector<MappingResultsVector_t> results;
  std::vector<std::string> text;
  std::string paf;
  MappingResultsVector_t one_to_one_records;   // skch_bm_one_to_one's working copy of the records, kept between calls
  std::vector<ContigInfo> one_to_one_queries;  // ... and its query names
  int32_t one_to_one_query_len = -1;
};
struct BmBatch {
  BmHandle *owner;
  ReadBatch batch;
};

void *skch_bm_create_ex(void *index_handle, float percentageIdentity, int device, int threads, int filter_mode, const int *devices,
                        int n_devices);
void *skch_bm_create(void *index_handle, float percentageIdentity, int device, int threads)
{
  return skch_bm_create_ex(index_handle, percentageIdentity, device, threads, filter::MAP, nullptr, 0);
}
/* filter_mode: 1 map, 2 one-to-one, 3 none (map_parameters.hpp); devices: the GPUs this one process drives (--devices) */
void *skch_bm_create_ex(void *index_handle, float percentageIdentity, int device, int threads, int filter_mode, const int *devices,
                        int n_devices)
{
  IndexHandle *ih = (IndexHandle *)index_handle;
  ih->p.percentageIdentity = percentageIdentity;
  ih->p.filterMode = filter_mode;
  ih->p.devices.assign(devices, devices + (devices ? n_devices : 0));
  ih->p.device = device;
  ih->p.threads = threads;
  ih->p.block_length = ih->p.segLength;
  ih->p.chain_gap = ih->p.segLength;
  if (const char *e = getenv("MM_SUB_BATCH_BASES")) ih->p.sub_batch_bases = strtoull(e, nullptr, 10); /* tuning hook */
  BmHandle *h = new BmHandle();
  h->ih = ih;
  h->bm = new BatchMapper(ih->p, *ih->sk);
  return h;
}
void skch_bm_destroy(void *hv)
{
  BmHandle *h = (BmHandle *)hv;
  if (h) { delete h->bm; delete h; }
}
mm_ctx *skch_bm_ctx(void *hv) { return ((BmHandle *)hv)->bm->context(); }

/* n_reads reads of read_len bases each in a pinned batch buffer (nibbles, every read at a multiple of 32 bases);
 * skch_bm_batch_fill packs the caller's text into it */
void *skch_bm_batch_create(void *hv, uint64_t n_reads, int32_t read_len, int32_t first_seq_counter)
{
  BmHandle *h = (BmHandle *)hv;
  BmBatch *b = new BmBatch();
  b->owner = h;
  const uint64_t A = ReadBatch::READ_ALIGN;
  b->batch.capacity = n_reads * (((uint64_t)read_len + A - 1) / A * A) + 64;
  b->batch.bases = h->bm->allocBases(b->batch.capacity);
  memset(b->batch.bases, 0x88, b->batch.capacity / 2 + 256);
  for (uint64_t i = 0; i < n_reads; i++)
    h->bm->addRead(b->batch, "read" + std::to_string(first_seq_counter + (int64_t)i), nullptr, read_len, (seqno_t)(first_seq_counter + i));
  return b;
}
/* what a reader does while it parses: `ascii` holds the batch's reads back to back as text (read r at r * read_len);
 * every read is packed to nibbles at its place in the batch, on `threads` threads. Returns the seconds it took. */
double skch_bm_batch_fill(void *bv, const char *ascii, int threads)
{
  BmBatch *b = (BmBatch *)bv;
  const auto t0 = std::chrono::steady_clock::now();
  const size_t n = b->batch.reads.size();
  std::atomic<size_t> next{0};
  auto work = [&]() {
    while (true) {
      const size_t lo = next.fetch_add(64);
      if (lo >= n) break;
      const size_t hi = std::min(n, lo + 64);
      for (size_t r = lo; r < hi; r++) {
        const ReadRec &rd = b->batch.reads[r];
        seqio::pack_bases(ascii + r * (size_t)rd.len, (uint64_t)rd.len, b->batch.nibbles(b->batch.segs[rd.first_seg].offset));
      }
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < std::max(1, threads); t++) pool.emplace_back(work);
  work();
  for (auto &th : pool) th.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
/* bytes of the batch that cross PCIe per mapping pass (nibbles of the used part of the buffer) */
uint64_t skch_bm_batch_bytes(void *bv) { return (((BmBatch *)bv)->batch.used + 1) / 2; }
/* the host packer by itself (tests): n text bases -> (n + 1) / 2 bytes */
void skch_pack_bases(const char *ascii, uint64_t n, uint8_t *out) { seqio::pack_bases(ascii, n, out); }
uint64_t skch_bm_batch_segments(void *bv, const mm_segment **segs)
{
  BmBatch *b = (BmBatch *)bv;
  if (segs) *segs = b->batch.segs.data();
  return b->batch.segs.size();
}
void skch_bm_batch_destroy(void *bv)
{
  BmBatch *b = (BmBatch *)bv;
  if (b) { b->owner->bm->freeBases(b->batch.bases); delete b; }
}

/* host buffers -> H2D -> K1/K2/K3 -> D2H -> host tail -> PAF text (kept in the handle). */
int skch_bm_map(void *hv, void *bv, uint64_t *paf_bytes, uint64_t *n_mapped_reads, uint64_t *n_mappings, float stage_ms[8],
                double *sec_device, double *sec_tail)
{
  BmHandle *h = (BmHandle *)hv;
  BmBatch *b = (BmBatch *)bv;
  const double d0 = h->bm->secondsDevice, t0 = h->bm->secondsHostTail;
  const auto tm0 = std::chrono::steady_clock::now();
  /* -f one-to-one: the per-read mappings are not final (the run-wide sweep follows, skch_bm_one_to_one): no text yet */
  const bool report_now = h->ih->p.filterMode != filter::ONETOONE;
  if (!report_now) h->text.clear();
  h->bm->mapBatch(b->batch, h->results, report_now ? &h->text : nullptr, nullptr);
  const auto tm1 = std::chrono::steady_clock::now();
  const uint64_t bytes = h->bm->lastTextBytes, mapped = h->bm->lastMappedReads, maps = h->bm->lastMappings; /* summed by the tail workers */
  if (getenv("MM_TRACE"))
    fprintf(stderr, "[trace] skch_bm_map: mapBatch %.1f ms, result summary %.1f ms\n",
            std::chrono::duration<double, std::milli>(tm1 - tm0).count(),
            std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tm1).count());
  if (paf_bytes) *paf_bytes = bytes;
  if (n_mapped_reads) *n_mapped_reads = mapped;
  if (n_mappings) *n_mappings = maps;
  if (stage_ms) memcpy(stage_ms, h->bm->lastStageMs, 8 * sizeof(float));
  if (sec_device) *sec_device = h->bm->secondsDevice - d0;
  if (sec_tail) *sec_tail = h->bm->secondsHostTail - t0;
  return 0;
}
/* the mappings of the last skch_bm_map as raw skch::MappingResult records (a POD, base_types.hpp:152-153): what a rank
 * hands to mm_records_allgather */
uint32_t skch_mapping_record_bytes() { return (uint32_t)sizeof(MappingResult); }
uint64_t skch_bm_results_raw(void *hv, void *out, uint64_t cap)
{
  BmHandle *h = (BmHandle *)hv;
  const size_t nr = h->results.size();
  uint64_t n = 0;
  for (auto &v : h->results) n += v.size();
  MappingResult *o = (MappingResult *)out;
  if (!o || n > cap) return n;
  /* every read's mappings are a heap block of their own: the copy is a million cache misses, spread over the host threads */
  const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, h->ih->p.threads), nr / 4096));
  std::vector<uint64_t> first((size_t)T + 1, 0);
  for (int t = 0; t < T; t++) {
    uint64_t c = 0;
    for (size_t r = nr * (size_t)t / (size_t)T; r < nr * (size_t)(t + 1) / (size_t)T; r++) c += h->results[r].size();
    first[(size_t)t + 1] = first[(size_t)t] + c;
  }
  auto work = [&](int t) {
    MappingResult *at = o + first[(size_t)t];
    for (size_t r = nr * (size_t)t / (size_t)T; r < nr * (size_t)(t + 1) / (size_t)T; r++) {
      const MappingResultsVector_t &v = h->results[r];
      if (!v.empty()) memcpy((void *)at, (const void *)v.data(), v.size() * sizeof(MappingResult));
      at += v.size();
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < T; t++) pool.emplace_back(work, t);
  work(0);
  for (auto &th : pool) th.join();
  return n;
}
/* -f one-to-one, the run-wide step (computeMap.hpp:358-405) over `n` raw records of any origin (one rank's, or all ranks'
 * after the all-gather): reference-axis plane sweep + sort + PAF text (kept in the handle, see skch_bm_paf_final). Queries
 * are the reads "read<i>" of query_len bases, i in [0, n_queries). Returns the number of mappings kept. */
uint64_t skch_bm_one_to_one(void *hv, const void *recs, uint64_t n, int32_t n_queries, int32_t query_len)
{
  BmHandle *h = (BmHandle *)hv;
  MappingResultsVector_t &all = h->one_to_one_records;
  all.assign((const MappingResult *)recs, (const MappingResult *)recs + n);
  std::vector<ContigInfo> &q = h->one_to_one_queries;
  if ((int32_t)q.size() != n_queries || h->one_to_one_query_len != query_len) {
    q.resize((size_t)n_queries);
    for (int32_t i = 0; i < n_queries; i++) q[(size_t)i] = ContigInfo{"read" + std::to_string(i), query_len};
    h->one_to_one_query_len = query_len;
  }
  h->paf.clear();
  h->bm->finalizeOneToOne(all, q, h->paf);
  return all.size();
}
const char *skch_bm_paf_final(void *hv, uint64_t *n)
{
  BmHandle *h = (BmHandle *)hv;
  if (n) *n = h->paf.size();
  return h->paf.c_str();
}
int skch_bm_device_count(void *hv) { return ((BmHandle *)hv)->bm->deviceCount(); }

/* the PAF text of the last skch_bm_map, concatenated in read order */
const char *skch_bm_paf(void *hv, uint64_t *n)
{
  BmHandle *h = (BmHandle *)hv;
  h->paf.clear();
  for (auto &t : h->text) h->paf += t;
  if (n) *n = h->paf.size();
  return h->paf.c_str();
}
/* flat copy of the last results (one row per mapping) for parity checks */
uint64_t skch_bm_results(void *hv, int32_t *out, uint64_t cap_rows)
{ /* row: querySeqId, queryStartPos, queryEndPos, refSeqId, refStartPos, refEndPos, strand, conservedSketches, blockLength, id*1e6 */
  BmHandle *h = (BmHandle *)hv;
  uint64_t n = 0;
  for (auto &v : h->results)
    for (auto &m : v) {
      if (n < cap_rows) {
        int32_t *r = out + n * 10;
        r[0] = m.querySeqId; r[1] = m.queryStartPos; r[2] = m.queryEndPos; r[3] = m.refSeqId; r[4] = m.refStartPos;
        r[5] = m.refEndPos; r[6] = m.strand; r[7] = m.conservedSketches; r[8] = m.blockLength; r[9] = (int32_t)(m.nucIdentity * 1e6f);
      }
      n++;
    }
  return n;
}

/* ---- input: the mapped-FASTA bulk reader against the line reader (tests) ----
 * returns -1 if FastaFile declines the file, else the number of records that differ (name, length or bases) between
 * the two readers; *n_records / *n_bases describe what the line reader saw */
int64_t skch_fasta_readers_diff(const char *path, int threads, uint64_t *n_records, uint64_t *n_bases)
{
  std::vector<std::pair<std::string, std::string>> ref;
  uint64_t bases = 0;
  if (!seqio::for_each_seq_in_file(path, {}, "", [&](const std::string &name, const std::string &seq) {
        ref.emplace_back(name, seq);
        bases += seq.size();
      }))
    return -2;
  if (n_records) *n_records = ref.size();
  if (n_bases) *n_bases = bases;
  seqio::FastaFile ff;
  if (!ff.open(path, threads)) return -1;
  const auto &recs = ff.records();
  int64_t bad = recs.size() > ref.size() ? (int64_t)(recs.size() - ref.size()) : (int64_t)(ref.size() - recs.size());
  for (size_t i = 0; i < std::min(recs.size(), ref.size()); i++) {
    std::string seq(recs[i].seq_len, '\0');
    ff.copy_bases(recs[i], &seq[0]);
    if (ff.name(recs[i]) != ref[i].first || seq != ref[i].second) { bad++; continue; }
    /* the packing variant of the same copy: nibbles straight from the file mapping == nibbles of the text */
    std::vector<uint8_t> a((recs[i].seq_len + 1) / 2 + 1, 0), b((recs[i].seq_len + 1) / 2 + 1, 0);
    ff.pack_bases(recs[i], a.data());
    seqio::pack_bases(seq.data(), seq.size(), b.data());
    if (recs[i].seq_len & 1) { a[recs[i].seq_len / 2] |= 0xF0; b[recs[i].seq_len / 2] |= 0xF0; }  /* unused nibble */
    if (a != b) bad++;
  }
  return bad;
}

/* ---- BGZF input (tests) ---- */

/* the host build of mm_inflate.h on one raw DEFLATE stream of exactly out_len inflated bytes: its mmi_status; *crc gets
 * the CRC-32 of the text when it inflated */
int skch_mmi_inflate(const uint8_t *comp, uint64_t comp_len, uint8_t *out, uint64_t out_len, uint32_t *crc)
{
  std::unique_ptr<mmi_tables> t(new mmi_tables());
  const int rc = mmi_inflate(comp, comp_len, out, out_len, *t, 0, 1);
  if (rc == MMI_OK && crc) {
    uint32_t tab[256];
    mmi_crc_table(tab, 0, 1);
    *crc = mmi_crc_finish(mmi_crc_share(tab, out, out_len, 0, 1), out_len);
  }
  return rc;
}

namespace {
/* the host inflater, made to report block `fail_at` of the whole file (counted across calls) as bad */
struct FailingInflater : seqio::HostInflater {
  int64_t fail_at, seen = 0;
  uint64_t calls = 0;
  explicit FailingInflater(int64_t f) : fail_at(f) {}
  int inflate(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc, uint64_t n,
              uint8_t *out, int64_t *bad_block, std::string &error) override
  {
    calls++;
    const int64_t first = seen;
    seen += (int64_t)n;
    if (fail_at >= first && fail_at < seen) {
      *bad_block = fail_at - first;
      error = "rejected by the test";
      return 1;
    }
    return HostInflater::inflate(comp, comp_off, out_off, crc, n, out, bad_block, error);
  }
};
thread_local std::string g_bgzf_error;
}  // namespace

const char *skch_bgzf_error() { return g_bgzf_error.c_str(); }

/* the text of a BGZF FASTA file as the windowed reader hands it over (windows of window_bytes, host inflater; block
 * fail_block reported bad, -1 = none): its length (the first cap bytes go to buf), -1 if the reader declines the file,
 * -3 on an error (skch_bgzf_error). *n_windows / *n_calls: windows handed over, inflater calls made. */
int64_t skch_bgzf_text(const char *path, uint64_t window_bytes, int threads, int64_t fail_block, uint8_t *buf, uint64_t cap,
                       uint64_t *n_windows, uint64_t *n_calls)
{
  seqio::BgzfFasta bz;
  if (!bz.open(path)) return -1;
  FailingInflater inf(fail_block);
  uint64_t n = 0, w = 0;
  const int rc = bz.for_each_window(inf, window_bytes, threads, [&](const seqio::FastaText &t) {
    if (n < cap) memcpy(buf + n, t.data(), std::min<uint64_t>(cap - n, t.size()));
    n += t.size();
    w++;
  });
  if (n_windows) *n_windows = w;
  if (n_calls) *n_calls = inf.calls;
  if (rc < 0) { g_bgzf_error = bz.error(); return -3; }
  return rc == 1 ? -1 : (int64_t)n;
}

/* everything gzread gives for a file (what the line reader reads): its length, the first cap bytes to buf */
int64_t skch_gzread_text(const char *path, uint8_t *buf, uint64_t cap)
{
  gzFile f = gzopen(path, "rb");
  if (!f) return -1;
  std::vector<char> b(1 << 20);
  uint64_t n = 0;
  int got;
  while ((got = gzread(f, b.data(), (unsigned)b.size())) > 0) {
    if (n < cap) memcpy(buf + n, b.data(), std::min<uint64_t>(cap - n, (uint64_t)got));
    n += (uint64_t)got;
  }
  gzclose(f);
  return (int64_t)n;
}

/* records of a BGZF FASTA file through the windowed reader (host inflater) against the line reader: -1 if the reader
 * declines the file, -3 on an error, else the number of records that differ in name, bases or nibbles */
int64_t skch_bgzf_readers_diff(const char *path, uint64_t window_bytes, int threads, uint64_t *n_records, uint64_t *n_bases)
{
  std::vector<std::pair<std::string, std::string>> ref;
  uint64_t bases = 0;
  if (!seqio::for_each_seq_in_file(path, {}, "", [&](const std::string &name, const std::string &seq) {
        ref.emplace_back(name, seq);
        bases += seq.size();
      }))
    return -2;
  if (n_records) *n_records = ref.size();
  if (n_bases) *n_bases = bases;
  seqio::BgzfFasta bz;
  if (!bz.open(path)) return -1;
  seqio::HostInflater inf;
  size_t i = 0;
  int64_t bad = 0;
  const int rc = bz.for_each_window(inf, window_bytes, threads, [&](const seqio::FastaText &t) {
    for (const seqio::FastaRecord &r : t.records()) {
      if (i >= ref.size()) { bad++; continue; }
      std::string seq(r.seq_len, '\0');
      t.copy_bases(r, &seq[0]);
      std::vector<uint8_t> a((r.seq_len + 1) / 2 + 1, 0), b((r.seq_len + 1) / 2 + 1, 0);
      t.pack_bases(r, a.data());
      seqio::pack_bases(seq.data(), seq.size(), b.data());
      if (r.seq_len & 1) { a[r.seq_len / 2] |= 0xF0; b[r.seq_len / 2] |= 0xF0; }
      if (t.name(r) != ref[i].first || seq != ref[i].second || a != b) bad++;
      i++;
    }
  });
  if (rc < 0) { g_bgzf_error = bz.error(); return -3; }
  if (rc == 1) return -1;
  return bad + (int64_t)(ref.size() - std::min(ref.size(), i));
}

/* skch_read_file_digest's digest through the windowed BGZF reader (host inflater); -1 if it declines the file */
int skch_bgzf_read_digest(const char *path, uint64_t window_bytes, int threads, uint64_t *n_records, uint64_t *n_bases, uint64_t *digest)
{
  uint64_t h = 1469598103934665603ULL, nr = 0, nb = 0;
  auto eat = [&h](const std::string &s) {
    for (unsigned char c : s) { h ^= c; h *= 1099511628211ULL; }
    h ^= 0xFF; h *= 1099511628211ULL;
  };
  seqio::BgzfFasta bz;
  if (!bz.open(path)) return -1;
  seqio::HostInflater inf;
  const int rc = bz.for_each_window(inf, window_bytes, threads, [&](const seqio::FastaText &t) {
    for (const auto &r : t.records()) {
      std::string seq(r.seq_len, '\0');
      t.copy_bases(r, &seq[0]);
      eat(t.name(r)); eat(seq); nr++; nb += seq.size();
    }
  });
  if (rc != 0) return rc == 1 ? -1 : -3;
  *n_records = nr; *n_bases = nb; *digest = h;
  return 0;
}

/* ---- FASTQ input (tests) ---- */

namespace {
thread_local std::string g_fastq_error;
}  // namespace

const char *skch_fastq_error() { return g_fastq_error.c_str(); }

/* an FNV-1a digest of every record's name, length and nibbles (seqio::pack_bases' format) of a file, in order: through
 * the line reader (window_bytes = 0), or through FastqReader in windows of window_bytes with the host build of
 * mm_fastq.h (device < 0) or mm_fastq on `device`. out[4]: records, bases, digest, windows handed over. Returns 0; -1
 * if FastqReader declines the file; -2 if the line reader cannot read it; -3 on an error (skch_fastq_error). */
int skch_fastq_digest(const char *path, uint64_t window_bytes, int threads, int device, uint64_t *out)
{
  uint64_t h = 1469598103934665603ULL, nr = 0, nb = 0, nw = 0;
  auto eat = [&h](const void *p, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) { h ^= ((const uint8_t *)p)[i]; h *= 1099511628211ULL; }
    h ^= 0xFF; h *= 1099511628211ULL;
  };
  auto record = [&](const char *name, uint64_t name_len, uint64_t len, const uint8_t *nib) {
    eat(name, name_len); eat(&len, 8); eat(nib, (len + 1) / 2);
    nr++; nb += len;
  };
  if (window_bytes == 0) {
    std::vector<uint8_t> nib;
    if (!seqio::for_each_seq_in_file(path, {}, "", [&](const std::string &name, const std::string &seq) {
          nib.assign((seq.size() + 1) / 2 + 1, 0);
          seqio::pack_bases(seq.data(), seq.size(), nib.data());
          record(name.data(), name.size(), seq.size(), nib.data());
        }))
      return -2;
  } else {
    seqio::FastqReader rd;
    if (!rd.open(path)) return -1;
    std::unique_ptr<seqio::FastqParser> p;
    if (device < 0) p.reset(new seqio::HostFastqParser());
    else p.reset(new seqio::DeviceFastqParser(device));
    const int rc = rd.for_each_window(*p, window_bytes, threads, [&](const mm_fastq_records &r) {
      for (uint64_t i = 0; i < r.n_records; i++)
        record(r.names + r.name_off[i], r.name_off[i + 1] - r.name_off[i], r.seq_len[i], r.nibbles + r.nib_off[i]);
      nw++;
    });
    if (rc != 0) { g_fastq_error = rd.error(); return -3; }
  }
  out[0] = nr; out[1] = nb; out[2] = h; out[3] = nw;
  return 0;
}

/* records, bases and an FNV-1a digest of every (name, sequence) pair of a file in order, through the line reader (bulk = 0)
 * or the memory-mapped bulk reader (bulk = 1; returns -1 when it declines the file): compared with the same digest taken
 * through the reference's own reader (oracle/_ref, refh_read_file_digest) */
int skch_read_file_digest(const char *path, int bulk, int threads, uint64_t *n_records, uint64_t *n_bases, uint64_t *digest)
{
  uint64_t h = 1469598103934665603ULL, nr = 0, nb = 0;
  auto eat = [&h](const std::string &s) {
    for (unsigned char c : s) { h ^= c; h *= 1099511628211ULL; }
    h ^= 0xFF; h *= 1099511628211ULL;
  };
  if (!bulk) {
    if (!seqio::for_each_seq_in_file(path, {}, "", [&](const std::string &name, const std::string &seq) {
          eat(name); eat(seq); nr++; nb += seq.size();
        }))
      return -2;
  } else {
    seqio::FastaFile ff;
    if (!ff.open(path, threads)) return -1;
    for (const auto &r : ff.records()) {
      std::string seq(r.seq_len, '\0');
      ff.copy_bases(r, &seq[0]);
      eat(ff.name(r)); eat(seq); nr++; nb += seq.size();
    }
  }
  *n_records = nr; *n_bases = nb; *digest = h;
  return 0;
}

/* Self-test of the run-wide one-to-one step (MapTail::finalizeOneToOne: sorts through (key, index) pairs, reference-axis
 * sweep per contig on `threads` threads, PAF text in slices) against the plain statement of computeMap.hpp:358-405 +
 * filter.hpp:333-394 (std::sort on the records, one serial sweep, one stream) on n random mappings full of ties.
 * One mapping in `span_every` covers its whole contig (0 = none: every contig is a sweep unit of its own, as with reads).
 * Returns the number of differing bytes of PAF text (0 = identical; -1 = different lengths). */
int64_t skch_one_to_one_selftest(int64_t n, uint64_t seed, int threads, int n_contigs, int n_queries, int span_every, double *sec_fast, double *sec_plain)
{
  Parameters p;
  p.filterMode = filter::ONETOONE; p.threads = threads; p.numMappingsForSegment = 1;
  std::vector<ContigInfo> meta, qmeta;
  std::vector<int> groups((size_t)n_contigs, 0);
  for (int i = 0; i < n_contigs; i++) meta.push_back(ContigInfo{"ctg" + std::to_string(i), 1000000});
  for (int i = 0; i < n_queries; i++) qmeta.push_back(ContigInfo{"read" + std::to_string(i), 20000});
  uint64_t x = seed * 0x9E3779B97F4A7C15ULL + 1;
  auto rnd = [&]() { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
  MappingResultsVector_t all((size_t)n);
  const float ids[6] = {0.95f, 0.96f, 0.97f, 0.9712f, 0.99f, 1.0f};
  for (auto &m : all) {
    memset(&m, 0, sizeof m);
    m.querySeqId = (seqno_t)(rnd() % (uint64_t)n_queries);
    m.queryLen = 20000;
    m.queryStartPos = (offset_t)((rnd() % 4) * 5000);
    m.queryEndPos = m.queryStartPos + 5000;
    m.refSeqId = (seqno_t)(rnd() % (uint64_t)n_contigs);
    m.refStartPos = (offset_t)((rnd() % 4000) * 250);  /* coarse grid: many equal starts */
    m.refEndPos = std::min<offset_t>(m.refStartPos + 4999 + (offset_t)(rnd() % 3) * 2500, 999999);
    if (span_every > 0 && rnd() % (uint64_t)span_every == 0) { m.refStartPos = 0; m.refEndPos = 999999; }  /* spans its contig: the linking case of the parallel sweep */
    m.nucIdentity = ids[rnd() % 6]; m.nucIdentityUpperBound = m.nucIdentity;
    m.blockLength = 5000; m.sketchSize = 20; m.conservedSketches = 15; m.strand = rnd() & 1 ? strnd::FWD : strnd::REV;
    m.kmerComplexity = 0.9; m.n_merged = 1;
  }
  std::sort(all.begin(), all.end(), [](const MappingResult &a, const MappingResult &b) { return a.querySeqId < b.querySeqId; });  /* read order */
  MapTail tail(p, meta, groups);
  /* plain */
  MappingResultsVector_t a = all;
  std::string paf_plain;
  auto t0 = std::chrono::steady_clock::now();
  {
    std::sort(a.begin(), a.end(), [](const MappingResult &l, const MappingResult &r) { return std::tie(l.refSeqId, l.refStartPos) < std::tie(r.refSeqId, r.refStartPos); });
    std::sort(a.begin(), a.end(), [](const MappingResult &l, const MappingResult &r) {
      return std::tie(l.queryStartPos, l.refSeqId, l.refStartPos) < std::tie(r.queryStartPos, r.refSeqId, r.refStartPos); });
    Filter::ref::filterMappings(a, meta, 0);
    std::sort(a.begin(), a.end(), [](const MappingResult &l, const MappingResult &r) {
      return std::tie(l.queryStartPos, l.refSeqId, l.refStartPos) < std::tie(r.queryStartPos, r.refSeqId, r.refStartPos); });
    std::sort(a.begin(), a.end(), [](const MappingResult &l, const MappingResult &r) {
      return std::tie(l.querySeqId, l.queryStartPos, l.refSeqId, l.refStartPos) < std::tie(r.querySeqId, r.queryStartPos, r.refSeqId, r.refStartPos); });
    std::ostringstream os;
    MapTail t2(p, meta, groups);
    t2.qmetadata = &qmeta;
    t2.formatMappings(a, "", os);
    paf_plain = os.str();
  }
  if (sec_plain) *sec_plain = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  MappingResultsVector_t b = all;
  std::string paf_fast;
  t0 = std::chrono::steady_clock::now();
  tail.finalizeOneToOne(b, qmeta, paf_fast);
  if (sec_fast) *sec_fast = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (paf_fast.size() != paf_plain.size()) return -1;
  int64_t diff = 0;
  for (size_t i = 0; i < paf_fast.size(); i++) diff += paf_fast[i] != paf_plain[i];
  return diff + (a.size() != b.size());
}

/* ---- host tail on caller-provided records ---- */
struct skch_tail_params {
  int32_t kmerSize, segLength, sketchSize, filterMode, numMappingsForSegment, numMappingsForShortSequence;
  int32_t block_length, chain_gap, mergeMappings, stage1_topANI_filter, keep_low_pct_id, skip_self, skip_prefix;
  int32_t prefix_delim, filterLengthMismatches, legacy_output, report_ANI_percentage;
  float percentageIdentity, ANIDiff, ANIDiffConf, kmerComplexityThreshold;
};

struct TailHandle {
  Parameters p;
  std::vector<ContigInfo> meta;
  std::vector<int> groups;
  MapTail *tail = nullptr;
  std::string text;
  MappingResultsVector_t last;
};

void *skch_tail_create(const skch_tail_params *tp, int n_contigs, const char **names, const int32_t *lens, const int32_t *groups)
{
  TailHandle *h = new TailHandle();
  Parameters &p = h->p;
  p.kmerSize = tp->kmerSize; p.segLength = tp->segLength; p.sketchSize = tp->sketchSize; p.filterMode = tp->filterMode;
  p.numMappingsForSegment = tp->numMappingsForSegment; p.numMappingsForShortSequence = tp->numMappingsForShortSequence;
  p.block_length = tp->block_length; p.chain_gap = tp->chain_gap; p.mergeMappings = tp->mergeMappings;
  p.stage1_topANI_filter = tp->stage1_topANI_filter; p.keep_low_pct_id = tp->keep_low_pct_id; p.skip_self = tp->skip_self;
  p.skip_prefix = tp->skip_prefix; p.prefix_delim = (char)tp->prefix_delim; p.filterLengthMismatches = tp->filterLengthMismatches;
  p.legacy_output = tp->legacy_output; p.report_ANI_percentage = tp->report_ANI_percentage;
  p.percentageIdentity = tp->percentageIdentity; p.ANIDiff = tp->ANIDiff; p.ANIDiffConf = tp->ANIDiffConf;
  p.kmerComplexityThreshold = tp->kmerComplexityThreshold;
  for (int i = 0; i < n_contigs; i++) {
    h->meta.push_back(ContigInfo{names[i], lens[i]});
    h->groups.push_back(groups ? groups[i] : 0);
  }
  h->tail = new MapTail(h->p, h->meta, h->groups);
  return h;
}

/* -f one-to-one, the run-wide step (MapTail::finalizeOneToOne) on caller-provided mappings in the flat record layout of the
 * checkers (oracle/mm_oracle_types.h orc_mapping: the members of skch::MappingResult as int32 / float / double), on `threads`
 * threads. No device involved: tests compare it with the reference's own statements of the step. Returns the mappings kept. */
struct skch_flat_mapping {
  int32_t queryLen, refStartPos, refEndPos, queryStartPos, queryEndPos, refSeqId, querySeqId, blockLength;
  float nucIdentity, nucIdentityUpperBound;
  int32_t sketchSize, conservedSketches, strand, approxMatches, n_merged, splitMappingId, discard, selfMapFilter;
  double kmerComplexity;
};
static void unflatten(const skch_flat_mapping &o, MappingResult &m)
{
  memset(&m, 0, sizeof m);
  m.queryLen = o.queryLen; m.refStartPos = o.refStartPos; m.refEndPos = o.refEndPos; m.queryStartPos = o.queryStartPos;
  m.queryEndPos = o.queryEndPos; m.refSeqId = o.refSeqId; m.querySeqId = o.querySeqId; m.blockLength = o.blockLength;
  m.nucIdentity = o.nucIdentity; m.nucIdentityUpperBound = o.nucIdentityUpperBound; m.sketchSize = o.sketchSize;
  m.conservedSketches = o.conservedSketches; m.strand = (strand_t)o.strand; m.approxMatches = o.approxMatches; m.n_merged = o.n_merged;
  m.splitMappingId = o.splitMappingId; m.discard = (uint8_t)o.discard; m.selfMapFilter = o.selfMapFilter != 0;
  m.kmerComplexity = o.kmerComplexity;
}
int64_t skch_tail_one_to_one(void *hv, const skch_flat_mapping *in, int64_t n, skch_flat_mapping *out, int32_t n_queries, int threads)
{
  TailHandle *h = (TailHandle *)hv;
  h->p.threads = threads;
  MappingResultsVector_t all((size_t)n);
  for (int64_t i = 0; i < n; i++) unflatten(in[i], all[(size_t)i]);
  std::vector<ContigInfo> q((size_t)n_queries);
  for (int32_t i = 0; i < n_queries; i++) q[(size_t)i] = ContigInfo{"q" + std::to_string(i), 0};
  h->tail->finalizeOneToOne(all, q, h->text);
  for (size_t i = 0; i < all.size(); i++) {
    const MappingResult &m = all[i];
    skch_flat_mapping &o = out[i];
    o.queryLen = m.queryLen; o.refStartPos = m.refStartPos; o.refEndPos = m.refEndPos; o.queryStartPos = m.queryStartPos;
    o.queryEndPos = m.queryEndPos; o.refSeqId = m.refSeqId; o.querySeqId = m.querySeqId; o.blockLength = m.blockLength;
    o.nucIdentity = m.nucIdentity; o.nucIdentityUpperBound = m.nucIdentityUpperBound; o.sketchSize = m.sketchSize;
    o.conservedSketches = m.conservedSketches; o.strand = m.strand; o.approxMatches = m.approxMatches; o.n_merged = m.n_merged;
    o.splitMappingId = m.splitMappingId; o.discard = m.discard; o.selfMapFilter = m.selfMapFilter; o.kmerComplexity = (double)m.kmerComplexity;
  }
  return (int64_t)all.size();
}
/* the PAF text of caller-provided mappings of one read (MapTail::formatMappings, the stream-free formatter the product
 * writes with), for comparison with the reference's own reportReadMappings (oracle/_ref, refh_report_mappings) */
const char *skch_tail_format(void *hv, const skch_flat_mapping *in, int64_t n, const char *queryName, uint64_t *n_bytes)
{
  TailHandle *h = (TailHandle *)hv;
  MappingResultsVector_t v((size_t)n);
  for (int64_t i = 0; i < n; i++) unflatten(in[i], v[(size_t)i]);
  h->text.clear();
  h->tail->formatMappings(v, queryName, h->text);
  if (n_bytes) *n_bytes = h->text.size();
  return h->text.c_str();
}

void skch_tail_destroy(void *hv)
{
  TailHandle *h = (TailHandle *)hv;
  if (h) { delete h->tail; delete h; }
}

/* mapModule's host part for ONE read whose fragments are segs[0..n_seg). Returns the PAF text. */
const char *skch_tail_map_read(void *hv, const char *name, int32_t len, int32_t seqCounter, int32_t refGroup,
                               const mm_segment *segs, const mm_segment_result *segRes, uint32_t n_seg,
                               const mm_l1_candidate *cands, const mm_l2_locus *loci, int32_t *n_out)
{
  TailHandle *h = (TailHandle *)hv;
  h->tail->segs = segs; h->tail->segRes = segRes; h->tail->cands = cands; h->tail->loci = loci;
  ReadRec rd;
  rd.name = name; rd.len = len; rd.seqCounter = seqCounter; rd.first_seg = 0; rd.n_seg = n_seg; rd.refGroup = refGroup;
  IdentityCache idc;
  idc.k = h->p.kmerSize; idc.ANIDiff = h->p.ANIDiff;
  h->last.clear();
  h->tail->mapRead(rd, idc, h->last);
  std::ostringstream os;
  h->tail->formatMappings(h->last, rd.name, os);
  h->text = os.str();
  if (n_out) *n_out = (int32_t)h->last.size();
  return h->text.c_str();
}

/* tail micro-benchmark (scripts/tail_perf.py): the host tail of n_reads reads, `iters` times over, on one thread.
 * The reads' records are back to back: read r owns fragments [seg_first[r], seg_first[r+1]) and its candidate / locus
 * indices are absolute. Returns seconds in mapRead and in formatMappings. */
void skch_tail_bench(void *hv, int32_t n_reads, const int32_t *read_len, const uint64_t *seg_first, const mm_segment *segs,
                     const mm_segment_result *segRes, const mm_l1_candidate *cands, const mm_l2_locus *loci, int iters,
                     double *sec_map, double *sec_format, uint64_t *n_mappings)
{
  TailHandle *h = (TailHandle *)hv;
  h->tail->segs = segs; h->tail->segRes = segRes; h->tail->cands = cands; h->tail->loci = loci;
  std::vector<ReadRec> reads((size_t)n_reads);
  for (int r = 0; r < n_reads; r++) {
    reads[r].name = "read" + std::to_string(r); reads[r].len = read_len[r]; reads[r].seqCounter = r;
    reads[r].first_seg = seg_first[r]; reads[r].n_seg = (uint32_t)(seg_first[r + 1] - seg_first[r]); reads[r].refGroup = -1;
  }
  IdentityCache idc;
  idc.k = h->p.kmerSize; idc.ANIDiff = h->p.ANIDiff;
  std::vector<MappingResultsVector_t> res((size_t)n_reads);
  std::ostringstream os;
  double tm = 0, tf = 0;
  uint64_t nm = 0;
  for (int it = 0; it < iters; it++) {
    auto t0 = std::chrono::steady_clock::now();
    for (int r = 0; r < n_reads; r++) { res[r].clear(); h->tail->mapRead(reads[r], idc, res[r]); }
    auto t1 = std::chrono::steady_clock::now();
    for (int r = 0; r < n_reads; r++) {
      if (res[r].empty()) continue;
      h->text.clear();
      h->tail->formatMappings(res[r], reads[r].name, h->text);
      nm += res[r].size();
    }
    auto t2 = std::chrono::steady_clock::now();
    tm += std::chrono::duration<double>(t1 - t0).count();
    tf += std::chrono::duration<double>(t2 - t1).count();
  }
  if (sec_map) *sec_map = tm;
  if (sec_format) *sec_format = tf;
  if (n_mappings) *n_mappings = nm;
}

int64_t skch_sort_selftest(int64_t n, uint64_t seed, int threads, int pattern, int64_t *heap_branches)
{
  return MapTail::sortSelftest(n, seed, threads, pattern, heap_branches);
}

/* the string formatter of the PAF lines against the stream formatter (the reference's own statement) on n random mappings,
 * in every output mode: returns the number of modes whose texts differ (0 = identical) */
int skch_format_selftest(int64_t n, uint64_t seed)
{
  std::mt19937_64 rng(seed);
  std::vector<ContigInfo> meta;
  for (int i = 0; i < 7; i++) meta.push_back(ContigInfo{"contig_" + std::to_string(i), 1000000 + i});
  std::vector<int> groups(meta.size(), 0);
  MappingResultsVector_t v((size_t)n);
  std::uniform_real_distribution<float> uf(0.0f, 1.0f);
  for (auto &m : v) {
    memset(&m, 0, sizeof(m));
    m.queryLen = (offset_t)(rng() % 200000); m.queryStartPos = (offset_t)(rng() % 100000); m.queryEndPos = m.queryStartPos + (offset_t)(rng() % 100000);
    m.refSeqId = (seqno_t)(rng() % meta.size()); m.refStartPos = (offset_t)(rng() % 1000000); m.refEndPos = m.refStartPos + (offset_t)(rng() % 100000);
    m.strand = (rng() & 1) ? strnd::FWD : strnd::REV;
    m.sketchSize = 1 + (int)(rng() % 1000); m.conservedSketches = (int)(rng() % (uint64_t)(m.sketchSize + 1)); m.blockLength = (int)(rng() % 100000);
    switch (rng() % 6) { /* identities: arbitrary floats, dyadic values (exact decimal ties), the extremes */
      case 0: m.nucIdentity = (float)(rng() % 129) / 128.0f; break;
      case 1: m.nucIdentity = (float)(rng() % 1025) / 1024.0f; break;
      case 2: m.nucIdentity = 1.0f; break;
      case 3: m.nucIdentity = uf(rng) * 1e-4f; break;
      default: m.nucIdentity = uf(rng);
    }
    switch (rng() % 4) {
      case 0: m.kmerComplexity = (long double)((double)(rng() % 1000) / 999.0); break;
      case 1: m.kmerComplexity = (long double)uf(rng); break;
      case 2: m.kmerComplexity = (long double)(((double)uf(rng) + (double)uf(rng) + (double)uf(rng)) / 3.0); break;
      default: m.kmerComplexity = 1.0L;
    }
  }
  int bad = 0;
  bad += (int)MapTail::realTextSelftest(n * 4, seed);  /* the number formatter alone, against snprintf("%g") */
  for (int mode = 0; mode < 8; mode++) {
    Parameters p;
    p.legacy_output = (mode & 1) != 0; p.report_ANI_percentage = (mode & 2) != 0; p.mergeMappings = (mode & 4) == 0;
    MapTail t(p, meta, groups);
    std::ostringstream os;
    t.formatMappingsStream(v, "query_name", os);
    std::string fast;
    t.formatMappings(v, "query_name", fast);
    if (os.str() != fast) bad++;
  }
  return bad;
}

/* --indexShards for the CPU tests: BatchMapper::planShards (first[n_shards + 1]; returns 0, or -1 with the reason in
 * skch_last_plan_error()) and the frequent seeds of the union of per-shard key counts (globalFrequentSeeds: writes the
 * ascending frequent hashes to out[cap], returns their number, or -1 when cap is too small) */
static thread_local std::string g_plan_error;
int skch_plan_shards(const uint64_t *len, const int32_t *group, int n_contigs, int by_group, int n_shards, int32_t *first)
{
  std::vector<int32_t> f;
  g_plan_error = BatchMapper::planShards(std::vector<uint64_t>(len, len + n_contigs), std::vector<int>(group, group + n_contigs),
                                         by_group != 0, n_shards, f);
  if (!g_plan_error.empty()) return -1;
  std::copy(f.begin(), f.end(), first);
  return 0;
}
const char *skch_last_plan_error() { return g_plan_error.c_str(); }
int64_t skch_global_frequent_seeds(int n_shards, const uint64_t *const *keys, const uint32_t *const *counts, const uint64_t *n,
                                   float kmer_pct_threshold, uint64_t *out, uint64_t cap, int32_t *threshold, uint64_t *n_unique)
{
  int t = 0;
  const std::vector<hash_t> f = globalFrequentSeeds(std::vector<const hash_t *>(keys, keys + n_shards),
                                                    std::vector<const uint32_t *>(counts, counts + n_shards),
                                                    std::vector<uint64_t>(n, n + n_shards), kmer_pct_threshold, t, *n_unique);
  *threshold = t;
  if (f.size() > cap) return -1;
  std::copy(f.begin(), f.end(), out);
  return (int64_t)f.size();
}

}  // extern "C"
