/*
 * mm_internal.h -- device-side data layout shared by the kernels and the C ABI (not installed).
 *
 * HBM layout (all arrays sub-allocated from ONE device arena, the "index blob", so that the whole
 * reference index can be moved to another GPU with a single broadcast):
 *
 *   minmer index, structure-of-arrays in reference order (seqId, wpos) (winSketch.hpp:102):
 *     idx_hash[n]  u64   idx_wpos[n] i32   idx_wend[n] i32   idx_strand[n] i8
 *     contig_start[n_contigs+1] u64   first index entry of each contig (seqId is implied)
 *   the same entries in "death order" -- per contig sorted by wpos_end (stable) -- for the L2 scan, which
 *   merges the insert stream (by wpos) with the delete stream (by wpos_end) instead of keeping a heap:
 *     idx2_hash[n] u64   idx2_wend[n] i32
 *   hash -> interval points (winSketch.hpp:100-101, ankerl map replaced by open addressing):
 *     tab[2^tab_log2] {u64 key, u64 val}; val = offset<<25 | count<<1 | is_freq; val==0 = empty
 *     pts[n_points] u64 = seqId<<33 | pos<<1 | (side==OPEN)        (8 B instead of 24 B)
 *   small tables: contig_len/name_id/group i32[n_contigs], cutoffs i32[], min_hits i32[]
 */
#ifndef MM_INTERNAL_H
#define MM_INTERNAL_H

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/mashmap_b200.h"
#include "mm_hash.h"

#define MM_TAB_EMPTY_VAL 0ULL
#define MM_VAL_OFF_SHIFT 25
#define MM_VAL_CNT_MASK 0xFFFFFFu

struct mm_tab_slot {
  uint64_t key;
  uint64_t val;
};

/* Offsets (bytes from blob start) of every array; lives at the start of the blob. */
struct mm_blob_header {
  uint64_t magic;
  uint64_t total_bytes;
  uint64_t n_minmers, n_keys, n_points;
  int32_t n_contigs, tab_log2, n_cutoffs, n_min_hits;
  uint64_t off_idx_hash, off_idx_wpos, off_idx_wend, off_idx_strand, off_contig_start;
  uint64_t off_idx2_hash, off_idx2_wend;
  uint64_t off_tab, off_pts;
  uint64_t off_contig_len, off_contig_name_id, off_contig_group;
  uint64_t off_cutoffs, off_min_hits;
};
#define MM_BLOB_MAGIC 0x4d4d4232303042ULL

/* Resolved device pointers, passed to kernels by value. */
struct mm_dev_index {
  const uint64_t *idx_hash;
  const int32_t *idx_wpos;
  const int32_t *idx_wend;
  const int8_t *idx_strand;
  const uint64_t *contig_start;
  const uint64_t *idx2_hash;
  const int32_t *idx2_wend;
  const mm_tab_slot *tab;
  const uint64_t *pts;
  const int32_t *contig_len;
  const int32_t *contig_name_id;
  const int32_t *contig_group;
  const int32_t *cutoffs;
  const int32_t *min_hits;
  uint64_t n_minmers;
  int32_t n_contigs;
  int32_t tab_log2;
  int32_t n_cutoffs;
  int32_t n_min_hits;
};

/* The per-batch counters in device memory: written by the kernels, zeroed by the host before K1 and read back by it as
 * one block (k_publish, mm_capi.cu: one word per lane of one warp). */
struct mm_counters {
  uint32_t cands_needed;        /* K2: candidates of the batch, including those past cand_cap                          */
  uint32_t l2_overflow;         /* K3: MM_L2_LOCI_OVERFLOW or MM_L2_LIVE_SET_OVERFLOW (the latter wins), 0 = none       */
  uint32_t scratch_overflow;    /* K2: the scratch pool is exhausted (1)                                               */
  uint32_t cand_overflow;       /* K2: candidates past cand_cap were dropped (1)                                       */
  unsigned long long pool_used; /* K2: bump pointer into the scratch pool, in u64 elements                              */
  uint32_t loci_needed;         /* K3 (k_l2, k_l2_long): end of the loci appended; the host sets where they start      */
  uint32_t l2_redo;             /* K3 (k_l2_scan): candidates flagged for the general kernel                           */
  uint32_t l1_cta_segments;     /* K2: segments the warp path handed to the CTA path (the CTA path's work count)       */
  uint32_t sketch_rejects;      /* K1: segments the fast sketch kernel handed to the general one (its work count)      */
  uint32_t _unused[6];
};
static_assert(offsetof(mm_counters, pool_used) == 16 && offsetof(mm_counters, pool_used) % 8 == 0,
              "the pool bump pointer is one 8-byte-aligned u64 atomic");
static_assert(sizeof(mm_counters) <= 16 * 4, "the counter block is read back by one warp, one word per lane");
constexpr uint32_t MM_L2_LOCI_OVERFLOW = 1;     /* the locus buffer is too small: grow it and run again */
constexpr uint32_t MM_L2_LIVE_SET_OVERFLOW = 2; /* more live index entries than the general kernel holds: an error */

/* Per-batch device buffers. */
struct mm_dev_batch {
  const uint8_t *bases;       /* ASCII bases (only when the batch came in as text), padded by 256 bytes          */
  const uint8_t *packed;      /* one nibble per base (2-bit code | 8 = not ACGT), base i in byte i/2, low nibble first; */
                              /* what the sketch kernel reads; padded by 256 bytes                                 */
  const mm_segment *segs;
  uint32_t n_segs;
  /* query sketches, slot seg*S + j (ascending hash); compacted in place by the L1 kernel      */
  uint64_t *sk_hash;
  uint64_t *sk_val;   /* lookup-table value of every sketch hash (written by the sketch kernels, mm_tab_lookup): */
                      /* 0 = absent; nullptr = no index, the sketch kernels skip the probe                      */
  int2 *sk_pos;               /* (first position, last position)                                */
  int8_t *sk_strand;
  int32_t *sk_votes;          /* optional (nullptr = not written; general sketch kernel only): the vote SUM of every     */
                              /* sketch slot, which the merge of a long fragment's pieces needs (sk_strand: its sign)   */
  mm_segment_result *seg_res;
  uint32_t *sk_reject;        /* work list of the general sketch kernel: segments the fast kernel handed over          */
  mm_l1_candidate *cands;
  uint32_t cand_cap;
  mm_l2_locus *loci;
  uint32_t loci_cap;
  mm_counters *counters;
  uint64_t *scratch;          /* global-memory work area for segments with many interval points:       */
                              /* one slice per CTA of the L1 grid, then a bump-allocated pool          */
  uint64_t scratch_slice;     /* u64 elements per CTA slice                                            */
  uint64_t scratch_pool_off;  /* first u64 element of the pool                                         */
  uint64_t scratch_cap;       /* total u64 elements                                                    */
  /* L2 work area */
  struct mm_l2_range *l2_ranges; /* per candidate: where its insert / delete streams are                */
  uint64_t *l2_rec_off;          /* per candidate (+1): first op record (exclusive prefix of the counts)   */
  uint2 *l2_recs;                /* op records {pos, info}                                                 */
  uint64_t l2_recs_cap;
  const uint32_t *l2_perm;       /* order in which k_l2_scan takes the candidates (nullptr = identity)        */
  uint32_t l2_loci_per_cand;     /* fixed locus slots per candidate in `loci`; overflow -> general kernel  */
  /* K2 of a contig-sharded index (--indexShards): MM_L1_BEST_ONLY writes each segment's sweep-#1 best to l1_best[seg]
   * and nothing else (no candidates, the sketch is not compacted); MM_L1_GIVEN_BEST takes the early return and the HG
   * raise from l1_best[seg] (the best over all shards) instead of its own sweep */
  int32_t *l1_best;
  /* MM_L1_GIVEN_BEST, fragments longer than seg_length: l1_after[seg] != 0 = a later shard has points of the segment. The
   * reference then tests this shard's last position group when its sweep moves on to that contig (:1026-1027) */
  const uint8_t *l1_after;
  int32_t l1_mode;
};
#define MM_L1_FULL 0
#define MM_L1_BEST_ONLY 1
#define MM_L1_GIVEN_BEST 2

/* insert stream = index entries [it0, it0+nI) (by wpos); delete stream = death-order entries [d0, d0+nD) */
struct mm_l2_range {
  uint64_t it0, d0;
  uint32_t nI, nD;
  int32_t next_wpos; /* wpos of entry it0+nI if it is on the same contig, else wpos of the last insert entry */
  uint32_t _pad;
};

/* op record info word */
#define MM_L2_SLOT_MASK 0xFFFFu   /* slot (1-based) of the hash in the query sketch; n+1 = above every query hash */
#define MM_L2_MATCH (1u << 16)    /* hash == query hash of that slot */
/* bits 17..18 of an insert record: q_strand * ref strand as 2-bit two's complement (-1, 0, +1) */

MM_HD uint32_t mm_tab_slot_of(uint64_t key, int log2)
{
  uint64_t x = (key ^ (key >> 29)) * 0x9E3779B97F4A7C15ULL;
  return (uint32_t)(x >> (64 - log2));
}

#ifdef __CUDACC__
/* the rest of a lookup whose first slot (key, val at `slot`) is already loaded: follow the linear-probe chain. Returns 0
 * when h is absent, else offset<<25 | count<<1 | isFreqSeed */
__device__ __forceinline__ uint64_t mm_tab_resolve(const mm_tab_slot *tab, int log2, uint64_t h, uint32_t slot, uint64_t key,
                                                   uint64_t val)
{
  const uint32_t tmask = (1u << log2) - 1u;
  while (val != MM_TAB_EMPTY_VAL && key != h) {
    slot = (slot + 1) & tmask;
    key = tab[slot].key;
    val = tab[slot].val;
  }
  return val;
}
__device__ __forceinline__ uint64_t mm_tab_lookup(const mm_tab_slot *tab, int log2, uint64_t h)
{
  const uint32_t slot = mm_tab_slot_of(h, log2);
  return mm_tab_resolve(tab, log2, h, slot, tab[slot].key, tab[slot].val);
}
#endif

/* launchers implemented in the .cu files; all return cudaError_t from the launch */
/* K1; where b.sk_val is set, every sketch hash written is also looked up in ix's table (K2's first step) */
cudaError_t mm_launch_sketch(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, cudaStream_t st, int sm_count,
                             int mode);
/* K1 for fragments longer than seg_length (mm_sketch.cu): the fragment was cut into pieces of at most seg_length bases
 * that overlap by kmer_size-1 (piece j starts at base j * (seg_length - kmer_size + 1)); the pieces were sketched by
 * mm_launch_sketch in mode 1 (general kernel) as segments [piece0, piece0 + n_pieces) of the same batch, with
 * b.sk_votes set. This merges the pieces of each long fragment into the fragment's own sketch slot. */
struct mm_long_frag {
  uint32_t seg;      /* the fragment's segment index: where its sketch goes          */
  uint32_t piece0;   /* segment index of its first piece                              */
  uint32_t n_pieces;
  uint32_t _pad;
};
size_t mm_sketch_long_tmp_bytes(uint64_t n_entries, uint32_t n_frags);
cudaError_t mm_launch_sketch_long_merge(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, const mm_long_frag *frags,
                                        const uint64_t *entry_off, uint32_t n_frags, uint32_t piece_base, uint64_t n_entries,
                                        void *tmp, size_t tmp_bytes, cudaStream_t st);
/* K0: ASCII -> nibbles (makeUpperCaseAndValidDNA as a format change); both buffers padded to a multiple of 16 bases */
cudaError_t mm_launch_pack_bases(const uint8_t *ascii, uint8_t *packed, uint64_t n_bases, cudaStream_t st, int sm_count);
cudaError_t mm_launch_l1(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b,
                         cudaStream_t st, int sm_count, uint32_t *slow_list, int use_warp_path, int *n_launched);
cudaError_t mm_launch_l2(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b,
                         uint32_t n_cands, cudaStream_t st, int sm_count);
/* K2 / K3 of the fragments longer than seg_length (windowLen > 0): the kernels above skip them. K3: one warp per
 * candidate of such a fragment, live hashes in a per-candidate open-addressing table of `table_slots[c]` slots at
 * `table_off[c]` in `table` (u64 words; sized by mm_launch_l2_long_ranges) */
cudaError_t mm_launch_l1_long(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, const mm_long_frag *longs,
                              uint32_t n_long, cudaStream_t st, int sm_count);
cudaError_t mm_launch_l2_long_ranges(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                     uint64_t *table_off, void *scan_tmp, size_t scan_tmp_bytes, cudaStream_t st);
cudaError_t mm_launch_l2_long(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                              const uint64_t *table_off, uint64_t *table, cudaStream_t st, int sm_count);
/* new L2: ranges -> (host reads the total) -> prep -> lane-per-candidate scan -> general kernel for overflow */
cudaError_t mm_launch_l2_ranges(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                void *scan_tmp, size_t scan_tmp_bytes, cudaStream_t st);
size_t mm_l2_scan_tmp_bytes(uint32_t n_cands);
size_t mm_l2_order_bytes(uint32_t n_cands);
cudaError_t mm_launch_l2_order(const mm_dev_batch &b, uint32_t n_cands, void *work, size_t work_bytes, uint32_t **perm, cudaStream_t st);
cudaError_t mm_launch_l2_prep(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                              cudaStream_t st, int sm_count);
cudaError_t mm_launch_l2_scan(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                              cudaStream_t st, int sm_count);
cudaError_t mm_launch_l2_overflow(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                  cudaStream_t st, int sm_count);
/* index image helpers (mm_index_build.cu): AoS -> device layouts, and back */
cudaError_t mm_upload_split_minmers(const mm_minmer *aos, uint64_t n, uint64_t *hash, int32_t *wpos, int32_t *wend,
                                    int8_t *strand, cudaStream_t st);
cudaError_t mm_upload_pack_points(const mm_ipoint *aos, uint64_t n, int32_t n_contigs, uint64_t *packed, uint32_t *err,
                                  cudaStream_t st);
cudaError_t mm_upload_build_table(const uint64_t *keys, const uint64_t *offs, const uint8_t *is_freq, uint64_t n_keys,
                                  mm_tab_slot *tab, int tab_log2, uint32_t *err, cudaStream_t st);
/* death-order arrays of the index (device-side sort) */
cudaError_t mm_build_death_order(const uint64_t *idx_hash, const int32_t *idx_wend, const uint64_t *contig_start,
                                 int32_t n_contigs, uint64_t n, uint64_t *idx2_hash, int32_t *idx2_wend, cudaStream_t st);
/* cnt[q] += number of entries of seq[0, n) equal to q */
cudaError_t mm_index_count_seq(uint64_t n, const int32_t *seq, unsigned long long *cnt, cudaStream_t st);
/* the n packed points back to skch::IntervalPoint, with the hash of the key whose list (keys, offs) holds each */
cudaError_t mm_index_unpack_points(uint64_t n, const uint64_t *pts, const uint64_t *keys, const uint64_t *offs, uint64_t n_keys,
                                   mm_ipoint *out, cudaStream_t st);
uint32_t mm_l1_grid_size(const mm_params &p, int sm_count);
int mm_sketch_kmer_supported(int k);
/* Shared memory one block may have on sm_90 (dynamic and static together), and the dynamic shared memory each kernel
 * whose size depends on the parameters is launched with; 0 where it cannot launch. The launchers and mm_params_check
 * both call these. */
constexpr size_t MM_SMEM_PER_BLOCK = 227 * 1024;
/* K1 (k_sketch_table) for (seg_length, sketch_size, kmer_size), its table and list capacities */
size_t mm_sketch_smem_bytes(int seg_length, int sketch_size, int kmer_size, int *table_cap, int *list_cap);
/* K2's general path (k_l1_cta, k_l1_long) */
size_t mm_l1_cta_smem(int sketch_size);
/* K3's general kernel (k_l2) and the live-set capacity it is launched with */
size_t mm_l2_general_smem(int sketch_size, int *live_cap);
/* K3 of the fragments longer than a segment (k_l2_long) */
size_t mm_l2_long_smem(int sketch_size);

#endif
