/*
 * mm_index_build.h -- device-side index builder (mm_index_build.cu), internal to libmashmap_b200.so.
 */
#ifndef MM_INDEX_BUILD_H
#define MM_INDEX_BUILD_H

#include <string>

#include "mm_devbuf.h"
#include "mm_internal.h"

/* the five columns of a set of minmer records, as kernels take them (by value) */
struct mm_rec_view {
  uint64_t *hash;
  int32_t *wpos, *wend, *seq;
  int8_t *strand;
};
struct mm_rec_cols {
  mm_devbuf<uint64_t> hash;
  mm_devbuf<int32_t> wpos, wend, seq;
  mm_devbuf<int8_t> strand;

  cudaError_t reserve(uint64_t n)
  {
    cudaError_t e;
    if ((e = hash.reserve(n)) != cudaSuccess || (e = wpos.reserve(n)) != cudaSuccess || (e = wend.reserve(n)) != cudaSuccess ||
        (e = seq.reserve(n)) != cudaSuccess || (e = strand.reserve(n)) != cudaSuccess)
      return e;
    return cudaSuccess;
  }
  void reset() { hash.reset(); wpos.reset(); wend.reset(); seq.reset(); strand.reset(); }
  mm_rec_view view() const { return mm_rec_view{hash.get(), wpos.get(), wend.get(), seq.get(), strand.get()}; }
};

/* device arrays the builder leaves behind (owned by the struct) */
struct mm_built_index {
  uint64_t n_minmers = 0, n_keys = 0, n_points = 0;
  /* minmerIndex after the frequent-seed drop, in reference order (seqId, wpos, wpos_end, emission order) */
  mm_rec_cols mi;
  /* on request (keep_unfiltered): minmerIndex BEFORE the drop, n_minmers_before_filter records -- what --saveIndex writes */
  mm_rec_cols mi_unfiltered;
  /* minmerPosLookupIndex, keys ascending: keys[n_keys], offs[n_keys + 1], pts[n_points] (packed, mm_pack_point), is_freq[n_keys] */
  mm_devbuf<uint64_t> keys, offs, pts; mm_devbuf<uint8_t> is_freq;
  mm_devbuf<uint32_t> counts; /* mm_freq_rule::COUNT_ONLY: the interval points of every key */
  int32_t freq_threshold = 0x7fffffff;
  /* statistics */
  uint64_t n_minmers_before_filter = 0;
  uint32_t n_chunks = 0, n_fixed_chunks = 0, fix_rounds = 0;
  uint32_t hist_min_count = 0, hist_max_count = 0;
  unsigned long long hist_min_keys = 0, hist_max_keys = 0;
  float ms_scan = 0, ms_post = 0, ms_lookup = 0;
};
/* Which keys the builder flags as frequent seeds and drops from minmerIndex.
 * OWN_THRESHOLD: the frequency threshold of kmer_pct_threshold `pct` over these contigs (an unsharded index).
 * The two passes over one shard of a contig-sharded index (--indexShards, DESIGN.md):
 * COUNT_ONLY: stop after Sketch::index and leave every distinct hash (ascending) in out->keys and its interval-point count
 *   in out->counts.
 * LISTED: d_freq[n_freq] (device, ascending) are the frequent hashes of the WHOLE reference: exactly those are flagged and
 *   dropped, in place of the builder's own threshold, and the listed hashes this shard does not contain are appended after
 *   its keys as frequent keys with no points. */
struct mm_freq_rule {
  enum { OWN_THRESHOLD, COUNT_ONLY, LISTED } mode;
  float pct;
  const uint64_t *d_freq;
  uint64_t n_freq;

  static mm_freq_rule own_threshold(float pct) { return mm_freq_rule{OWN_THRESHOLD, pct, nullptr, 0}; }
  static mm_freq_rule count_only() { return mm_freq_rule{COUNT_ONLY, 0.f, nullptr, 0}; }
  static mm_freq_rule listed(const uint64_t *d_freq, uint64_t n_freq) { return mm_freq_rule{LISTED, 0.f, d_freq, n_freq}; }
};
/* d_seq: the contigs as text, back to back, on the device (readable up to h_contig_off[n_contigs]); a contig of length 0
 * gets no records (so a shard keeps the global seqIds of its contigs). keep_unfiltered: leave the records before the
 * frequent-seed drop in out->mi_unfiltered instead of freeing them. Returns MM_OK or MM_E* */
int mm_build_index_device(const mm_params &p, const uint8_t *d_seq, const uint64_t *h_contig_off, int32_t n_contigs,
                          const mm_freq_rule &rule, bool keep_unfiltered, cudaStream_t st, int sm_count, mm_built_index *out,
                          std::string &err);
/* The same index from a minmer list instead of text (a loaded --saveIndex file): aos[n] (on the device if aos_on_device,
 * else in host memory) is taken as the records before the frequent-seed drop, and the stages after the window scan run
 * on it (the lookup, and the frequency filter of mm_freq_rule::own_threshold(kmer_pct_threshold)). Every record is
 * checked first, before anything is indexed by its seqId: a seqId outside [0, n_contigs), a record before the one in
 * front of it in (seqId, wpos) order, or a negative wpos / wpos_end is refused with MM_EINVAL, err naming the first such
 * record. */
int mm_build_index_from_records(const mm_minmer *aos, int aos_on_device, uint64_t n, int32_t n_contigs, float kmer_pct_threshold,
                                bool keep_unfiltered, cudaStream_t st, mm_built_index *out, std::string &err);
/* SoA -> AoS: the records of `in` as mm_minmer (_pad = 0) in out[n] (device) */
cudaError_t mm_pack_minmers(const mm_rec_cols &in, uint64_t first, uint64_t n, mm_minmer *out, cudaStream_t st);

#endif
