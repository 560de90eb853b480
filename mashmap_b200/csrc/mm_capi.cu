/*
 * mm_capi.cu -- implementation of the C ABI declared in include/mashmap_b200.h.
 *
 * Owns the device context: the index blob (one arena, see mm_internal.h), the per-batch buffers,
 * the stream and the stage timers, and drives K1 (mm_sketch.cu) -> K2 (mm_l1.cu) -> K3 (mm_l2.cu).
 * There is no CPU implementation behind any entry point: without a usable sm_90 device every call
 * fails with MM_ENODEVICE.
 */
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "mm_devbuf.h"
#include "mm_index_build.h"
#include "mm_internal.h"
#include <chrono>

static thread_local std::string g_create_error;

struct mm_ctx {
  int device = -1;
  int sm_count = 0;
  mm_params params{};
  cudaStream_t stream = nullptr;
  std::string error;
  uint64_t launches = 0;
  uint64_t diag[8] = {0}; /* mm_ctx_diag: how often the rare paths ran (cumulative) */

  /* index blob: the context's own (own_blob), or a view of the one of share_src */
  mm_devbuf<unsigned char> own_blob;
  unsigned char *blob = nullptr;
  uint64_t blob_bytes = 0;
  bool blob_ready = false;
  mm_blob_header hdr{};
  mm_dev_index ix{};
  std::vector<int32_t> cutoffs, min_hits;

  /* batch */
  mm_devbuf<uint8_t> d_bases; uint64_t n_bases = 0;
  mm_devbuf<uint8_t> d_packed; /* nibbles */
  mm_built_index built{}; /* lookup arrays of an index built on the device, kept for mm_index_download (keep_lookup) */
  bool built_kept = false;
  bool batch_is_ascii = false; /* the resident batch came in as text: K0 (pack) runs in front of K1 */
  cudaEvent_t ev_pack = nullptr;
  float pack_ms = 0;
  mm_devbuf<mm_segment> d_segs; uint64_t n_segs = 0;
  /* fragments longer than seg_length: K1 runs over d_work_segs = the caller's n_segs segments (a long one replaced by its
   * first piece), then the n_work - n_segs pieces the long ones are cut into; d_long lists them (n_long) */
  mm_devbuf<mm_segment> d_work_segs;
  uint64_t n_work = 0; uint32_t n_long = 0; uint64_t long_entries = 0;
  mm_devbuf<uint64_t> d_sk_hash, d_sk_val; mm_devbuf<int2> d_sk_pos; mm_devbuf<int8_t> d_sk_strand;
  mm_devbuf<mm_segment_result> d_seg_res;
  mm_devbuf<uint32_t> d_sk_reject;
  int sk_mode = 0; /* 0 = fast sketch kernel + general kernel over its rejects; 1 = general kernel only (MM_SKETCH_TABLE=1) */
  /* fragments longer than seg_length: vote sums of the pieces, the fragment list and the merge area (K1); the live-table
   * offsets, the scan's work area and the live tables (K3) */
  mm_devbuf<int32_t> d_sk_votes;
  mm_devbuf<mm_long_frag> d_long;
  mm_devbuf<uint64_t> d_long_off;
  mm_devbuf<unsigned char> d_long_tmp;
  mm_devbuf<uint64_t> d_l2_long_off;
  mm_devbuf<unsigned char> d_long_scan_tmp;
  mm_devbuf<uint64_t> d_long_table;
  mm_devbuf<mm_l1_candidate> d_cands;
  mm_devbuf<mm_l2_locus> d_loci;
  mm_devbuf<uint32_t> d_counters;
  bool blocking_wait = false;       /* MM_BLOCKING_WAIT=1: host waits block on an event instead of spinning (experiment) */
  cudaEvent_t ev_wait = nullptr;
  const mm_ctx *share_src = nullptr; /* mm_ctx_share_index: the context whose index image this one reads */
  mm_phase_hook hook = nullptr;
  void *hook_user = nullptr;
  uint32_t *h_pub = nullptr; /* pinned, device-mapped: kernels publish counters here (no copy engine involved) */
  mm_devbuf<uint64_t> d_scratch; uint64_t scratch_slice = 0; uint64_t scratch_pool = 0;
  uint32_t l1_grid = 0;
  uint64_t n_cands = 0, n_loci = 0;
  /* the L2 stream path's own work areas: the ranges, the record offsets, the scan's and the candidate ordering's
   * (mm_launch_l2_order) temporaries are sized together, by d_l2_ranges' capacity; then the operation records */
  mm_devbuf<mm_l2_range> d_l2_ranges; mm_devbuf<uint64_t> d_l2_rec_off;
  mm_devbuf<unsigned char> d_scan_tmp, d_l2_order;
  mm_devbuf<uint2> d_l2_recs;
  mm_devbuf<uint32_t> d_l1_slow;
  int l1_warp = 1; /* 1 = warp-per-segment fast path + CTA path for big segments; 0 = CTA path only (MM_L1_CTA=1) */
  int l2_mode = 1; /* 1 = stream kernels (mm_l2_stream.cu), 0 = general kernel only (MM_L2_GENERAL=1) */
  bool batch_mapped = false;

  cudaEvent_t ev[10]{};
  float stage_ms[8]{};
};

namespace {

int fail(mm_ctx *c, int code, const char *fmt, ...)
{
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->error = buf; else g_create_error = buf;
  return code;
}

#define CU(c, call)                                                                              \
  do {                                                                                           \
    cudaError_t e_ = (call);                                                                     \
    if (e_ != cudaSuccess)                                                                       \
      return fail(c, e_ == cudaErrorMemoryAllocation ? MM_ENOMEM : MM_ECUDA, "%s: %s", #call,    \
                  cudaGetErrorString(e_));                                                       \
  } while (0)

uint64_t align_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

void resolve_index(mm_ctx *c)
{
  const mm_blob_header &h = c->hdr;
  unsigned char *b = c->blob;
  mm_dev_index &ix = c->ix;
  ix.idx_hash = (const uint64_t *)(b + h.off_idx_hash);
  ix.idx_wpos = (const int32_t *)(b + h.off_idx_wpos);
  ix.idx_wend = (const int32_t *)(b + h.off_idx_wend);
  ix.idx_strand = (const int8_t *)(b + h.off_idx_strand);
  ix.contig_start = (const uint64_t *)(b + h.off_contig_start);
  ix.idx2_hash = (const uint64_t *)(b + h.off_idx2_hash);
  ix.idx2_wend = (const int32_t *)(b + h.off_idx2_wend);
  ix.tab = (const mm_tab_slot *)(b + h.off_tab);
  ix.pts = (const uint64_t *)(b + h.off_pts);
  ix.contig_len = (const int32_t *)(b + h.off_contig_len);
  ix.contig_name_id = (const int32_t *)(b + h.off_contig_name_id);
  ix.contig_group = (const int32_t *)(b + h.off_contig_group);
  ix.cutoffs = (const int32_t *)(b + h.off_cutoffs);
  ix.min_hits = (const int32_t *)(b + h.off_min_hits);
  ix.n_minmers = h.n_minmers;
  ix.n_contigs = h.n_contigs;
  ix.tab_log2 = h.tab_log2;
  ix.n_cutoffs = h.n_cutoffs;
  ix.n_min_hits = h.n_min_hits;
}

constexpr uint64_t TABLE_REGION_BYTES = 64 * 1024; /* room reserved for each of cutoffs / min_hits */

int write_tables(mm_ctx *c)
{
  if (!c->blob || c->cutoffs.empty() || c->min_hits.empty()) return MM_OK;
  if (c->cutoffs.size() * 4 > TABLE_REGION_BYTES || c->min_hits.size() * 4 > TABLE_REGION_BYTES)
    return fail(c, MM_EINVAL, "lookup tables too large");
  c->hdr.n_cutoffs = (int32_t)c->cutoffs.size();
  c->hdr.n_min_hits = (int32_t)c->min_hits.size();
  CU(c, cudaMemcpyAsync(c->blob + c->hdr.off_cutoffs, c->cutoffs.data(), c->cutoffs.size() * 4, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(c->blob + c->hdr.off_min_hits, c->min_hits.data(), c->min_hits.size() * 4, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(c->blob, &c->hdr, sizeof(c->hdr), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  resolve_index(c);
  return MM_OK;
}

/* the context has no index afterwards: its own image is freed, a shared one is no longer read */
void drop_index(mm_ctx *c)
{
  c->own_blob.reset();
  c->blob = nullptr; c->blob_bytes = 0; c->blob_ready = false; c->share_src = nullptr;
}

/* an index upload or build that returns before its image is complete leaves the context with no index */
struct image_guard {
  mm_ctx *c;
  ~image_guard() { if (!c->blob_ready) drop_index(c); }
};

/* lays out the index image for these counts (mm_internal.h) and allocates it as the context's own */
int begin_image(mm_ctx *c, uint64_t n_mi, uint64_t n_keys, uint64_t n_points, int32_t n_contigs)
{
  mm_blob_header h{};
  h.magic = MM_BLOB_MAGIC;
  h.n_minmers = n_mi; h.n_keys = n_keys; h.n_points = n_points;
  h.n_contigs = n_contigs; h.tab_log2 = 4;
  while ((1ULL << h.tab_log2) < 2 * n_keys + 2) h.tab_log2++;
  uint64_t o = align_up(sizeof(mm_blob_header), 256);
  auto place = [&](uint64_t bytes) { uint64_t at = o; o = align_up(o + bytes, 256); return at; };
  h.off_idx_hash = place((n_mi + 1) * 8);
  h.off_idx_wpos = place((n_mi + 1) * 4);
  h.off_idx_wend = place((n_mi + 1) * 4);
  h.off_idx_strand = place(n_mi + 1);
  h.off_contig_start = place(((uint64_t)n_contigs + 1) * 8);
  h.off_idx2_hash = place((n_mi + 1) * 8);
  h.off_idx2_wend = place((n_mi + 1) * 4);
  h.off_tab = place((1ULL << h.tab_log2) * sizeof(mm_tab_slot));
  h.off_pts = place((n_points + 1) * 8);
  h.off_contig_len = place((uint64_t)n_contigs * 4);
  h.off_contig_name_id = place((uint64_t)n_contigs * 4);
  h.off_contig_group = place((uint64_t)n_contigs * 4);
  h.off_cutoffs = place(TABLE_REGION_BYTES);
  h.off_min_hits = place(TABLE_REGION_BYTES);
  h.total_bytes = o;
  if (c->own_blob.reserve(o) != cudaSuccess)
    return fail(c, MM_ENOMEM, "cannot allocate the index image (%llu bytes)", (unsigned long long)o);
  c->blob = c->own_blob.get(); c->blob_bytes = o; c->hdr = h;
  return MM_OK;
}

/* Completes the image begun by begin_image once the caller has put the SoA index and the packed points in place (and
 * flagged bad points in d_err, bit 1): contig starts, death order, lookup table from the device key lists, contig
 * tables, header. Then the context reads it. */
int finish_image(mm_ctx *c, const std::vector<uint64_t> &cstart, const uint64_t *d_keys, const uint64_t *d_offs,
                 const uint8_t *d_freq, uint32_t *d_err, const int32_t *contig_len, const int32_t *contig_name_id,
                 const int32_t *contig_group)
{
  const mm_blob_header &h = c->hdr;
  const size_t n_contigs = (size_t)h.n_contigs;
  CU(c, cudaMemcpyAsync(c->blob + h.off_contig_start, cstart.data(), cstart.size() * 8, cudaMemcpyHostToDevice, c->stream));
  /* the same entries per contig in wpos_end order (device sort), for the L2 stream merge */
  CU(c, mm_build_death_order((const uint64_t *)(c->blob + h.off_idx_hash), (const int32_t *)(c->blob + h.off_idx_wend),
                             (const uint64_t *)(c->blob + h.off_contig_start), h.n_contigs, h.n_minmers,
                             (uint64_t *)(c->blob + h.off_idx2_hash), (int32_t *)(c->blob + h.off_idx2_wend), c->stream));
  /* open-addressing table, filled on the device */
  CU(c, cudaMemsetAsync(c->blob + h.off_tab, 0, (1ULL << h.tab_log2) * sizeof(mm_tab_slot), c->stream));
  CU(c, mm_upload_build_table(d_keys, d_offs, d_freq, h.n_keys, (mm_tab_slot *)(c->blob + h.off_tab), h.tab_log2, d_err, c->stream));
  uint32_t err = 0;
  CU(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  if (err & 1) return fail(c, MM_EINVAL, "an interval point has a bad seqId or a negative position");
  if (err & 2) return fail(c, MM_EINVAL, "a key has no or too many (>= 2^24) interval points, or offsets overflow");
  if (err & 4) return fail(c, MM_EINVAL, "duplicate key in the lookup index");
  CU(c, cudaMemcpyAsync(c->blob + h.off_contig_len, contig_len, n_contigs * 4, cudaMemcpyHostToDevice, c->stream));
  std::vector<int32_t> tmp(n_contigs, -1);
  CU(c, cudaMemcpyAsync(c->blob + h.off_contig_name_id, contig_name_id ? contig_name_id : tmp.data(), n_contigs * 4, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream)); /* tmp is rewritten below */
  std::fill(tmp.begin(), tmp.end(), 0);
  CU(c, cudaMemcpyAsync(c->blob + h.off_contig_group, contig_group ? contig_group : tmp.data(), n_contigs * 4, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(c->blob, &c->hdr, sizeof(c->hdr), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  resolve_index(c);
  c->blob_ready = true;
  return write_tables(c);
}

/* wait for the context's stream. Default: cudaStreamSynchronize (spins, lowest latency). With MM_BLOCKING_WAIT=1 the
 * thread sleeps on a blocking event instead -- for hosts with fewer usable CPUs than pipeline threads (DESIGN section 9). */
cudaError_t wait_stream(mm_ctx *c)
{
  if (!c->blocking_wait) return cudaStreamSynchronize(c->stream);
  const cudaError_t e = cudaEventRecord(c->ev_wait, c->stream);
  return e != cudaSuccess ? e : cudaEventSynchronize(c->ev_wait);
}

int check_ready(mm_ctx *c)
{
  if (!c) return MM_EINVAL;
  if (c->share_src) { /* follow the owner: its image may have been replaced since (new upload / adopted blob / new tables) */
    const mm_ctx *s = c->share_src;
    if (c->blob != s->blob || c->blob_bytes != s->blob_bytes || c->hdr.n_cutoffs != s->hdr.n_cutoffs ||
        c->hdr.n_min_hits != s->hdr.n_min_hits || c->blob_ready != s->blob_ready) {
      c->blob = s->blob; c->blob_bytes = s->blob_bytes; c->hdr = s->hdr; c->blob_ready = s->blob_ready;
      resolve_index(c);
    }
  }
  if (!c->blob_ready) return fail(c, MM_ESTATE, "reference index not uploaded");
  if (c->hdr.n_cutoffs <= 0 || c->hdr.n_min_hits <= 0) return fail(c, MM_ESTATE, "threshold tables not uploaded");
  return MM_OK;
}

/* A segment may be longer than seg_length (an unsplit query, windowLen > 0), up to the length at which the reference's
 * (len - k + 1) * 2 (an int, computeMap.hpp:831) overflows. */
int validate_segments(mm_ctx *c, const mm_segment *segs, uint64_t n_segs, uint64_t n_bases)
{
  if (n_segs >= (1ULL << 31)) return fail(c, MM_EINVAL, "too many segments in one batch");
  for (uint64_t i = 0; i < n_segs; i++) {
    const mm_segment &s = segs[i];
    if (s.length < 1 || (int64_t)s.length - c->params.kmer_size + 1 >= (1LL << 30))
      return fail(c, MM_EINVAL, "segment %llu: length %d outside [1, 2^30 + kmer_size - 2] (the reference computes "
                  "(length - k + 1) * 2 in an int)", (unsigned long long)i, s.length);
    if (s.offset + (uint64_t)s.length > n_bases) return fail(c, MM_EINVAL, "segment %llu exceeds the base buffer", (unsigned long long)i);
  }
  return MM_OK;
}

/* batch buffers that do not depend on the input format */
int prepare_batch_buffers(mm_ctx *c, uint64_t n_bases, uint64_t n_segs)
{
  /* nibbles: n_bases/2 rounded up to 8-byte groups of 16 bases, + 256 so that the 16-byte-granular bulk copies of the
   * sketch kernel never leave the allocation */
  const uint64_t pbytes = (n_bases + 15) / 16 * 8, packed_had = c->d_packed.capacity();
  CU(c, c->d_packed.reserve(pbytes + 256));
  if (c->d_packed.capacity() != packed_had) CU(c, cudaMemsetAsync(c->d_packed.get(), 0x88, c->d_packed.capacity(), c->stream));
  CU(c, c->d_segs.reserve(n_segs + 1));
  const uint64_t n = n_segs * (uint64_t)c->params.sketch_size + 1;
  CU(c, c->d_sk_hash.reserve(n));
  CU(c, c->d_sk_val.reserve(n));
  CU(c, c->d_sk_pos.reserve(n));
  CU(c, c->d_sk_strand.reserve(n));
  CU(c, c->d_seg_res.reserve(n_segs + 1));
  CU(c, c->d_sk_reject.reserve(n_segs + 1));
  CU(c, c->d_counters.reserve(16));
  return MM_OK;
}

/* experiment (MM_UPLOAD_KERNEL=<CTAs>): the host -> device copy done by a few CTAs that read the pinned host buffer
 * through its unified address (PCIe reads issued by SMs) instead of by the copy engine */
__global__ void __launch_bounds__(256) k_copy_from_host(uint4 *dst, const uint4 *src, uint64_t n16)
{
  const uint64_t stride = (uint64_t)gridDim.x * 256ULL;
  uint64_t i = (uint64_t)blockIdx.x * 256ULL + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    const uint4 a = __ldcs(src + i), b = __ldcs(src + i + stride), c = __ldcs(src + i + 2 * stride), d = __ldcs(src + i + 3 * stride);
    dst[i] = a; dst[i + stride] = b; dst[i + 2 * stride] = c; dst[i + 3 * stride] = d;
  }
  for (; i < n16; i += stride) dst[i] = __ldcs(src + i);
}

/* host -> device copy of `bytes` bytes, in <= 16 MiB pieces when a phase hook is installed (MM_PHASE_UPLOAD_CHUNK) */
int copy_in(mm_ctx *c, uint8_t *dst, const void *src, uint64_t bytes)
{
  static const int skip_after = getenv("MM_SKIP_H2D") ? atoi(getenv("MM_SKIP_H2D")) : 0; /* experiment: timing without the copies */
  static const int copy_ctas = getenv("MM_UPLOAD_KERNEL") ? atoi(getenv("MM_UPLOAD_KERNEL")) : 0;
  static std::atomic<int> calls{0};
  if (skip_after > 0 && calls.fetch_add(1) >= skip_after) return MM_OK;
  auto one = [&](uint8_t *d, const uint8_t *s_, uint64_t n) -> cudaError_t {
    if (copy_ctas > 0 && ((uintptr_t)d % 16 == 0) && ((uintptr_t)s_ % 16 == 0)) {
      const uint64_t n16 = n / 16;
      if (n16) k_copy_from_host<<<copy_ctas, 256, 0, c->stream>>>((uint4 *)d, (const uint4 *)s_, n16);
      if (n % 16) return cudaMemcpyAsync(d + n16 * 16, s_ + n16 * 16, n % 16, cudaMemcpyHostToDevice, c->stream);
      return cudaGetLastError();
    }
    return cudaMemcpyAsync(d, s_, n, cudaMemcpyHostToDevice, c->stream);
  };
  if (!c->hook) {
    CU(c, one(dst, (const uint8_t *)src, bytes));
    return MM_OK;
  }
  const uint64_t CH = 16ULL << 20;
  for (uint64_t at = 0; at < bytes; at += CH) {
    const uint64_t n = std::min(CH, bytes - at);
    c->hook(c->hook_user, MM_PHASE_UPLOAD_CHUNK, 1);
    cudaError_t e = one(dst + at, (const uint8_t *)src + at, n);
    if (e == cudaSuccess) e = wait_stream(c);
    c->hook(c->hook_user, MM_PHASE_UPLOAD_CHUNK, 0);
    CU(c, e);
  }
  return MM_OK;
}

/* packed != 0: `bases` holds nibbles (mm_batch_upload_packed).
 * A fragment longer than seg_length is sketched as pieces of at most seg_length bases that overlap by k-1 (piece j starts
 * at base j * (seg_length - k + 1)); the sketch kernels see the caller's segments with the pieces appended and merged into
 * the fragment's own slot afterwards (mm_launch_sketch_long_merge, mm_sketch.cu); that slot is sketched as a copy of the
 * first piece meanwhile (the merge overwrites it). Everything after K1 sees the caller's segments. */
int upload_batch(mm_ctx *c, const void *bases, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs, int packed)
{
  int rc = validate_segments(c, segs, n_segs, n_bases);
  if (rc) return rc;
  CU(c, cudaSetDevice(c->device));
  /* a failed upload leaves an empty batch, not counts that its buffers may no longer hold */
  c->n_segs = c->n_work = 0;
  c->n_long = 0;
  c->batch_mapped = false;
  const uint64_t S = (uint64_t)c->params.sketch_size;
  const int L = c->params.seg_length, step = L - c->params.kmer_size + 1;
  std::vector<mm_segment> work;
  std::vector<mm_long_frag> longs;
  std::vector<uint64_t> entry_off(1, 0);
  for (uint64_t i = 0; i < n_segs; i++) {
    const mm_segment &s = segs[i];
    if (s.length <= L) continue;
    if (work.empty()) work.assign(segs, segs + n_segs);
    const uint32_t n_pieces = (uint32_t)(((int64_t)s.length - c->params.kmer_size + step) / step);
    longs.push_back(mm_long_frag{(uint32_t)i, (uint32_t)work.size(), n_pieces, 0});
    for (uint32_t p = 0; p < n_pieces; p++) {
      mm_segment q = s;
      q.offset += (uint64_t)p * (uint64_t)step;
      q.length = (int32_t)std::min<int64_t>(L, (int64_t)s.length - (int64_t)p * step);
      work.push_back(q);
    }
    work[i].length = L;
    entry_off.push_back(entry_off.back() + (uint64_t)n_pieces * S);
  }
  const uint64_t n_work = longs.empty() ? n_segs : work.size();
  if (n_work >= (1ULL << 31) || entry_off.back() >= (1ULL << 32))
    return fail(c, MM_EINVAL, "too many segments in one batch after cutting the long fragments into pieces");
  if ((rc = prepare_batch_buffers(c, n_bases, n_work))) return rc;
  if (!longs.empty()) {
    CU(c, c->d_work_segs.reserve(n_work));
    CU(c, cudaMemcpyAsync(c->d_work_segs.get(), work.data(), n_work * sizeof(mm_segment), cudaMemcpyHostToDevice, c->stream));
    CU(c, c->d_sk_votes.reserve(c->d_sk_hash.capacity()));
    CU(c, c->d_long.reserve(longs.size()));
    CU(c, c->d_long_off.reserve(entry_off.size()));
    CU(c, c->d_long_tmp.reserve(mm_sketch_long_tmp_bytes(entry_off.back(), (uint32_t)longs.size())));
    CU(c, cudaMemcpyAsync(c->d_long.get(), longs.data(), longs.size() * sizeof(mm_long_frag), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(c->d_long_off.get(), entry_off.data(), entry_off.size() * 8, cudaMemcpyHostToDevice, c->stream));
  }
  CU(c, cudaEventRecord(c->ev[6], c->stream));
  if (packed) {
    const uint64_t pbytes = (n_bases + 1) / 2;
    if ((rc = copy_in(c, c->d_packed.get(), bases, pbytes))) return rc;
    CU(c, cudaMemsetAsync(c->d_packed.get() + pbytes, 0x88, 64, c->stream));
    if (n_bases & 1) { /* the unused high nibble of the last byte is whatever the caller had there: irrelevant (never a k-mer) */ }
  } else {
    CU(c, c->d_bases.reserve(n_bases + 256));
    if ((rc = copy_in(c, c->d_bases.get(), bases, n_bases))) return rc;
    CU(c, cudaMemsetAsync(c->d_bases.get() + n_bases, 'N', 256, c->stream));
  }
  CU(c, cudaMemcpyAsync(c->d_segs.get(), segs, n_segs * sizeof(mm_segment), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaEventRecord(c->ev[7], c->stream));
  if (!longs.empty()) CU(c, cudaStreamSynchronize(c->stream)); /* work / longs / entry_off are about to go */
  c->n_bases = n_bases;
  c->n_segs = n_segs;
  c->n_work = n_work;
  c->n_long = (uint32_t)longs.size();
  c->long_entries = entry_off.back();
  c->batch_is_ascii = !packed;
  return MM_OK;
}

/* K0 in front of K1 when the resident batch is text */
int launch_pack_if_ascii(mm_ctx *c)
{
  if (!c->batch_is_ascii) { c->pack_ms = 0; return MM_OK; }
  CU(c, mm_launch_pack_bases(c->d_bases.get(), c->d_packed.get(), c->n_bases, c->stream, c->sm_count));
  c->launches++;
  return MM_OK;
}

mm_dev_batch make_batch(mm_ctx *c);

/* K1 over the resident batch: the sketch kernels over the caller's segments and the pieces of the long fragments, then
 * the merge of the pieces. probe: the kernels also look every hash of the caller's segments up in the index's table
 * (sk_val, read by K2); the pieces' own hashes never are */
int launch_sketch_all(mm_ctx *c, bool probe)
{
  mm_dev_batch b = make_batch(c);
  if (c->n_long) b.segs = c->d_work_segs.get();
  if (!probe) b.sk_val = nullptr;
  CU(c, mm_launch_sketch(c->params, c->ix, b, c->stream, c->sm_count, c->sk_mode));
  c->launches += c->sk_mode ? 1 : 2;
  if (c->n_long) {
    /* the pieces: general kernel (it writes the vote sums the merge needs), then the merge */
    const uint64_t S = (uint64_t)c->params.sketch_size, n0 = c->n_segs;
    mm_dev_batch bp = b;
    bp.segs = c->d_work_segs.get() + n0; bp.n_segs = (uint32_t)(c->n_work - n0);
    bp.sk_hash = b.sk_hash + n0 * S; bp.sk_pos = b.sk_pos + n0 * S; bp.sk_strand = b.sk_strand + n0 * S;
    bp.sk_votes = c->d_sk_votes.get() + n0 * S; bp.seg_res = b.seg_res + n0; bp.sk_val = nullptr;
    CU(c, mm_launch_sketch(c->params, c->ix, bp, c->stream, c->sm_count, 1));
    b.sk_votes = c->d_sk_votes.get();
    CU(c, mm_launch_sketch_long_merge(c->params, c->ix, b, c->d_long.get(), c->d_long_off.get(), c->n_long, (uint32_t)n0,
                                      c->long_entries, c->d_long_tmp.get(), c->d_long_tmp.capacity(), c->stream));
    c->launches += 3; /* pieces, prep, merge (the segmented sort is a library call, not counted) */
  }
  return MM_OK;
}

mm_dev_batch make_batch(mm_ctx *c)
{
  mm_dev_batch b{};
  b.bases = c->d_bases.get(); b.packed = c->d_packed.get(); b.segs = c->d_segs.get(); b.n_segs = (uint32_t)c->n_segs;
  b.sk_hash = c->d_sk_hash.get(); b.sk_val = c->d_sk_val.get(); b.sk_pos = c->d_sk_pos.get(); b.sk_strand = c->d_sk_strand.get();
  b.seg_res = c->d_seg_res.get(); b.sk_reject = c->d_sk_reject.get();
  b.cands = c->d_cands.get(); b.cand_cap = (uint32_t)std::min<uint64_t>(c->d_cands.capacity(), 0xffffffffu);
  b.loci = c->d_loci.get(); b.loci_cap = (uint32_t)std::min<uint64_t>(c->d_loci.capacity(), 0xffffffffu);
  b.counters = c->d_counters.get();
  b.scratch = c->d_scratch.get(); b.scratch_slice = c->scratch_slice; b.scratch_pool_off = c->scratch_pool;
  b.scratch_cap = c->d_scratch.capacity();
  b.l2_ranges = c->d_l2_ranges.get(); b.l2_rec_off = c->d_l2_rec_off.get();
  b.l2_recs = c->d_l2_recs.get(); b.l2_recs_cap = c->d_l2_recs.capacity();
  b.l2_loci_per_cand = 2;
  return b;
}

int ensure_scratch(mm_ctx *c, uint64_t pool_elems)
{
  if (c->l1_grid == 0) {
    c->l1_grid = mm_l1_grid_size(c->params, c->sm_count);
    if (c->l1_grid == 0) return fail(c, MM_ECUDA, "cannot size the L1 grid");
  }
  const uint64_t slice = 3ULL << 16; /* 65536 points per CTA slice */
  c->scratch_slice = slice;
  c->scratch_pool = slice * c->l1_grid;
  CU(c, c->d_scratch.reserve(c->scratch_pool + pool_elems));
  return MM_OK;
}

/* Small device->host readbacks do not go through a copy engine: a DMA queued while another context's batch upload
 * (hundreds of MB) is in flight waits for it. A one-warp kernel stores the words into pinned, device-mapped host memory. */
__global__ void k_publish(const uint32_t *__restrict__ src, volatile uint32_t *dst, int n)
{
  if ((int)threadIdx.x < n) dst[threadIdx.x] = src[threadIdx.x];
  __threadfence_system();
}
__global__ void k_set_u32(uint32_t *dst, uint32_t v) { *dst = v; }
/* cudaMemsetAsync of a few words may be executed by a copy engine too: zero them with a kernel */
__global__ void k_zero_words(uint32_t *dst, int n) { if ((int)threadIdx.x < n) dst[threadIdx.x] = 0; }
#define ZERO_WORDS(c, ptr, n) do { k_zero_words<<<1, 32, 0, (c)->stream>>>((uint32_t *)(ptr), (n)); (c)->launches++; CU((c), cudaGetLastError()); } while (0)

int read_words(mm_ctx *c, const void *dev, uint32_t *out, int n_words)
{
  k_publish<<<1, 32, 0, c->stream>>>((const uint32_t *)dev, c->h_pub, n_words);
  c->launches++;
  CU(c, cudaGetLastError());
  CU(c, wait_stream(c));
  for (int i = 0; i < n_words; i++) out[i] = c->h_pub[i];
  return MM_OK;
}
#define RD(c, dev, out, n) do { int rc__ = read_words((c), (dev), (out), (n)); if (rc__) return rc__; } while (0)

/* returned by run_l2_stream when its own work areas cannot be allocated: the general kernel maps the batch instead */
constexpr int L2_STREAM_NO_ROOM = 1;

/* K3 fast path (mm_l2_stream.cu): ranges+scan -> records -> lane-per-candidate scan -> general kernel for the
 * candidates that need more locus slots. */
int run_l2_stream(mm_ctx *c, uint32_t *h_cnt)
{
  const uint64_t nc = c->n_cands;
  const uint32_t LPC = 2;
  CU(c, cudaEventRecord(c->ev[3], c->stream));
  if (nc == 0) {
    CU(c, cudaEventRecord(c->ev[4], c->stream));
    CU(c, wait_stream(c));
    c->n_loci = 0;
    return MM_OK;
  }
  if (nc + 1 > c->d_l2_ranges.capacity()) {
    const uint64_t want = nc + nc / 8 + 1024;
    if (c->d_l2_ranges.reserve(want) || c->d_l2_rec_off.reserve(want + 1) ||
        c->d_scan_tmp.reserve(mm_l2_scan_tmp_bytes((uint32_t)want) + 256) ||
        c->d_l2_order.reserve(mm_l2_order_bytes((uint32_t)want))) {
      c->d_l2_ranges.reset(); /* its capacity stands for all four */
      return L2_STREAM_NO_ROOM;
    }
  }
  if (c->d_loci.capacity() < nc * LPC + 1024) CU(c, c->d_loci.reserve(nc * LPC + nc / 8 + 4096));
  mm_dev_batch b = make_batch(c);
  const auto tk0 = std::chrono::steady_clock::now();
  ZERO_WORDS(c, c->d_l2_rec_off.get() + nc, 2);
  CU(c, mm_launch_l2_ranges(c->params, c->ix, b, (uint32_t)nc, c->d_scan_tmp.get(), c->d_scan_tmp.capacity(), c->stream));
  uint64_t total = 0;
  RD(c, c->d_l2_rec_off.get() + nc, (uint32_t *)&total, 2);
  const auto tk1 = std::chrono::steady_clock::now();
  c->stage_ms[6] = std::chrono::duration<float, std::milli>(tk1 - tk0).count(); /* host view: ranges + scan + readback */
  /* the scan's record readers run up to 2 * RING_CHUNKS + 2 records past a stream's end */
  if (total + 64 > c->d_l2_recs.capacity() && c->d_l2_recs.reserve(total + total / 16 + 1024)) return L2_STREAM_NO_ROOM;
  for (int attempt = 0; attempt < 4; attempt++) {
    b = make_batch(c);
    ZERO_WORDS(c, c->d_counters.get() + 1, 1);
    ZERO_WORDS(c, c->d_counters.get() + 6, 2);
    /* the record-preparation kernel is the bandwidth-bound one: no PCIe upload next to it (MM_PHASE_L2) */
    {
      struct phase_guard { /* the hook is always closed, whatever fails in between */
        mm_ctx *c; bool open;
        explicit phase_guard(mm_ctx *cc) : c(cc), open(cc->hook != nullptr) { if (open) c->hook(c->hook_user, MM_PHASE_L2, 1); }
        void close() { if (open) { c->hook(c->hook_user, MM_PHASE_L2, 0); open = false; } }
        ~phase_guard() { close(); }
      } guard(c);
      CU(c, cudaEventRecord(c->ev[8], c->stream));
      CU(c, mm_launch_l2_prep(c->params, c->ix, b, (uint32_t)nc, c->stream, c->sm_count));
      CU(c, cudaEventRecord(c->ev[9], c->stream));
      if (guard.open && c->blocking_wait) CU(c, cudaEventRecord(c->ev_wait, c->stream));
      uint32_t *perm = nullptr;
      CU(c, mm_launch_l2_order(b, (uint32_t)nc, c->d_l2_order.get(), c->d_l2_order.capacity(), &perm, c->stream));
      b.l2_perm = perm;
      CU(c, mm_launch_l2_scan(c->params, c->ix, b, (uint32_t)nc, c->stream, c->sm_count));
      /* the scan is already queued behind it: waiting for the end of the preparation kernel costs no bubble */
      if (guard.open) CU(c, cudaEventSynchronize(c->blocking_wait ? c->ev_wait : c->ev[9]));
    }
    c->launches += 4; /* own kernels: ranges, prep, order keys, scan (the prefix sum and the sort are library calls, not counted) */
    RD(c, c->d_counters.get(), h_cnt, 16);
    uint64_t extent = nc * LPC;
    if (h_cnt[7] > 0) { /* candidates with more than LPC loci: general kernel, loci appended after the fixed slots */
      c->diag[MM_DIAG_L2_GENERAL_CANDS] += h_cnt[7];
      const uint32_t base = (uint32_t)extent;
      k_set_u32<<<1, 1, 0, c->stream>>>(c->d_counters.get() + 6, base);
      c->launches++;
      CU(c, mm_launch_l2_overflow(c->params, c->ix, b, (uint32_t)nc, c->stream, c->sm_count));
      c->launches += 1;
      RD(c, c->d_counters.get(), h_cnt, 16);
      if (h_cnt[1] == 2) return fail(c, MM_ECUDA, "L2 live-set overflow in the general kernel");
      if (h_cnt[1] == 1 || h_cnt[6] > c->d_loci.capacity()) { /* grow and redo prep+scan+overflow */
        c->diag[MM_DIAG_L2_LOCI_REGROW]++;
        CU(c, c->d_loci.reserve((uint64_t)h_cnt[6] + h_cnt[6] / 4 + 1024));
        continue;
      }
      extent = h_cnt[6];
    }
    CU(c, cudaEventRecord(c->ev[4], c->stream));
    CU(c, wait_stream(c));
    cudaEventElapsedTime(&c->stage_ms[6], c->ev[8], c->ev[9]); /* k_l2_prep */
    cudaEventElapsedTime(&c->stage_ms[7], c->ev[9], c->ev[4]); /* k_l2_scan (+ overflow kernel) */
    c->n_loci = extent;
    return MM_OK;
  }
  return fail(c, MM_ECUDA, "locus buffer kept overflowing");
}

/* K3 of the candidates of fragments longer than seg_length (k_l2_long, mm_l2.cu), after the loci of the others, which end
 * at c->n_loci: live-table sizes -> offsets -> (host reads the total) -> the scans, appending at counters[6]. Records
 * ev[4] again at its end. */
int run_l2_long(mm_ctx *c, uint32_t *h_cnt)
{
  const uint64_t nc = c->n_cands;
  if (c->n_long == 0 || nc == 0) return MM_OK;
  CU(c, c->d_l2_long_off.reserve(nc + 1));
  CU(c, c->d_long_scan_tmp.reserve(mm_l2_scan_tmp_bytes((uint32_t)nc) + 256));
  mm_dev_batch b = make_batch(c);
  CU(c, mm_launch_l2_long_ranges(c->params, c->ix, b, (uint32_t)nc, c->d_l2_long_off.get(), c->d_long_scan_tmp.get(),
                                 c->d_long_scan_tmp.capacity(), c->stream));
  c->launches++;
  uint64_t words = 0;
  RD(c, c->d_l2_long_off.get() + nc, (uint32_t *)&words, 2);
  if (words == 0) return MM_OK;
  CU(c, c->d_long_table.reserve(words));
  for (int attempt = 0; attempt < 4; attempt++) {
    b = make_batch(c);
    ZERO_WORDS(c, c->d_counters.get() + 1, 1);
    k_set_u32<<<1, 1, 0, c->stream>>>(c->d_counters.get() + 6, (uint32_t)c->n_loci);
    CU(c, mm_launch_l2_long(c->params, c->ix, b, (uint32_t)nc, c->d_l2_long_off.get(), c->d_long_table.get(), c->stream,
                            c->sm_count));
    c->launches += 2;
    CU(c, cudaEventRecord(c->ev[4], c->stream));
    RD(c, c->d_counters.get(), h_cnt, 16);
    if (h_cnt[1] == 1 || h_cnt[6] > c->d_loci.capacity()) { /* a bigger locus buffer that keeps the loci already there, then again */
      c->diag[MM_DIAG_L2_LOCI_REGROW]++;
      CU(c, c->d_loci.reserve_keep((uint64_t)h_cnt[6] + h_cnt[6] / 4 + 1024, c->n_loci, c->stream));
      continue;
    }
    c->n_loci = h_cnt[6];
    return MM_OK;
  }
  return fail(c, MM_ECUDA, "locus buffer kept overflowing");
}

/* K3 by the general kernel (mm_l2.cu), retried alone if the locus buffer is too small (it is idempotent) */
int run_l2_general(mm_ctx *c, uint32_t *h_cnt)
{
  for (int attempt = 0; attempt < 4; attempt++) {
    const mm_dev_batch b = make_batch(c);
    ZERO_WORDS(c, c->d_counters.get() + 1, 1);
    ZERO_WORDS(c, c->d_counters.get() + 6, 2);
    CU(c, cudaEventRecord(c->ev[3], c->stream));
    CU(c, mm_launch_l2(c->params, c->ix, b, (uint32_t)c->n_cands, c->stream, c->sm_count));
    CU(c, cudaEventRecord(c->ev[4], c->stream));
    if (c->n_cands) c->launches += 1;
    RD(c, c->d_counters.get(), h_cnt, 16);
    if (h_cnt[1] == 2) return fail(c, MM_ECUDA, "L2 live-set overflow: the reference index has more than "
                                   "sketch_size+64 overlapping minmer windows at one position");
    if (h_cnt[1] == 1 || h_cnt[6] > c->d_loci.capacity()) {
      CU(c, c->d_loci.reserve((uint64_t)h_cnt[6] + h_cnt[6] / 4 + 1024));
      continue;
    }
    c->n_loci = h_cnt[6];
    return MM_OK;
  }
  return fail(c, MM_ECUDA, "locus buffer kept overflowing");
}

/* K1 -> K2 -> K3 on the resident batch, growing output buffers and retrying on overflow */
int run_pipeline(mm_ctx *c)
{
  int rc = check_ready(c);
  if (rc) return rc;
  CU(c, cudaSetDevice(c->device));
  c->batch_mapped = false;
  const uint64_t n_segs = c->n_segs;
  CU(c, c->d_cands.reserve(2 * n_segs + 1024));
  CU(c, c->d_loci.reserve(2 * c->d_cands.capacity()));
  uint64_t pool0 = 32ULL << 20; /* interval points the bump pool holds at first (grown on demand below) */
  if (const char *e = getenv("MM_L1_POOL_ELEMS")) pool0 = std::max<uint64_t>(1024, strtoull(e, nullptr, 10)); /* tests: force the regrow path */
  if ((rc = ensure_scratch(c, c->d_scratch ? c->d_scratch.capacity() - c->scratch_pool : pool0))) return rc;
  if (c->d_l1_slow.capacity() < n_segs + 1) CU(c, c->d_l1_slow.reserve(n_segs + n_segs / 8 + 1024));

  uint32_t h_cnt[16];
  for (int attempt = 0; attempt < 6; attempt++) {
    mm_dev_batch b = make_batch(c);
    ZERO_WORDS(c, c->d_counters.get(), 16);
    CU(c, cudaEventRecord(c->ev[0], c->stream));
    if ((rc = launch_pack_if_ascii(c))) return rc;
    CU(c, cudaEventRecord(c->ev_pack, c->stream));
    if ((rc = launch_sketch_all(c, true))) return rc;
    CU(c, cudaEventRecord(c->ev[1], c->stream));
    int l1_launches = 0;
    CU(c, mm_launch_l1(c->params, c->ix, b, c->stream, c->sm_count, c->d_l1_slow.get(), c->l1_warp, &l1_launches));
    if (c->n_long) { /* windowLen > 0: k_l1_long (mm_l1.cu), after the general path (it reuses its scratch slices) */
      CU(c, mm_launch_l1_long(c->params, c->ix, b, c->d_long.get(), c->n_long, c->stream, c->sm_count));
      l1_launches++;
    }
    CU(c, cudaEventRecord(c->ev[2], c->stream));
    c->launches += (uint64_t)l1_launches;
    RD(c, c->d_counters.get(), h_cnt, 16);
    const uint64_t need_cands = h_cnt[0];
    bool retry = false;
    c->diag[MM_DIAG_L1_CTA_SEGMENTS] += h_cnt[8];
    c->diag[MM_DIAG_SKETCH_GENERAL_SEGMENTS] += h_cnt[9];
    if (h_cnt[3] || need_cands > c->d_cands.capacity()) {
      c->diag[MM_DIAG_CAND_REGROW]++;
      CU(c, c->d_cands.reserve(need_cands + need_cands / 4 + 1024));
      retry = true;
    }
    if (h_cnt[2]) { /* scratch pool exhausted: quadruple it */
      c->diag[MM_DIAG_L1_POOL_REGROW]++;
      if ((rc = ensure_scratch(c, (c->d_scratch.capacity() - c->scratch_pool) * 4))) return rc;
      retry = true;
    }
    if (retry) continue;
    c->n_cands = need_cands;
    /* K3: the stream kernels, or the general kernel where they are off or their own work areas do not fit */
    rc = c->l2_mode == 1 ? run_l2_stream(c, h_cnt) : L2_STREAM_NO_ROOM;
    if (rc == L2_STREAM_NO_ROOM) rc = run_l2_general(c, h_cnt);
    if (rc || (rc = run_l2_long(c, h_cnt))) return rc;
    if (c->batch_is_ascii) cudaEventElapsedTime(&c->pack_ms, c->ev[0], c->ev_pack);
    cudaEventElapsedTime(&c->stage_ms[0], c->ev_pack, c->ev[1]);
    cudaEventElapsedTime(&c->stage_ms[1], c->ev[1], c->ev[2]);
    cudaEventElapsedTime(&c->stage_ms[2], c->ev[3], c->ev[4]);
    cudaEventElapsedTime(&c->stage_ms[5], c->ev[0], c->ev[4]); /* first launch -> last kernel end, incl. host gaps */
    c->diag[MM_DIAG_LONG_FRAGMENTS] += c->n_long;
    c->batch_mapped = true;
    return MM_OK;
  }
  return fail(c, MM_ECUDA, "candidate/scratch buffers kept overflowing");
}

/* the first mapping kernel that cannot be launched for these sizes, or nullptr if all of them can */
const char *kernel_that_does_not_fit(int seg_length, int sketch_size, int kmer_size)
{
  if (mm_sketch_smem_bytes(seg_length, sketch_size, kmer_size, nullptr, nullptr) == 0) return "the sketch kernel (K1)";
  if (mm_l1_cta_smem(sketch_size) == 0) return "the general L1 kernel (K2)";
  if (mm_l2_general_smem(sketch_size, nullptr) == 0) return "the general L2 kernel (K3)";
  if (mm_l2_long_smem(sketch_size) == 0) return "the L2 kernel of fragments longer than a segment (K3)";
  return nullptr;
}

} // namespace

extern "C" {

int mm_params_check(const mm_params *params)
{
  if (!params) return fail(nullptr, MM_EINVAL, "null params");
  if (!mm_sketch_kmer_supported(params->kmer_size))
    return fail(nullptr, MM_EINVAL, "k-mer size %d is not compiled in (8..32)", params->kmer_size);
  if (params->sketch_size < 1 || params->seg_length < params->kmer_size)
    return fail(nullptr, MM_EINVAL, "bad sketch_size / seg_length");
  const int L = params->seg_length, S = params->sketch_size, k = params->kmer_size;
  const char *stage = kernel_that_does_not_fit(L, S, k);
  if (!stage) return MM_OK;
  /* the largest sketch size that fits: every size is smaller than S, and acceptance falls off once in S */
  int lo = 0, hi = S; /* lo fits (or is 0), hi does not */
  while (hi - lo > 1) {
    const int mid = lo + (hi - lo) / 2;
    if (kernel_that_does_not_fit(L, mid, k)) hi = mid; else lo = mid;
  }
  if (lo == 0)
    return fail(nullptr, MM_EINVAL, "seg_length %d / sketch_size %d exceed the shared-memory budget of %s; no sketch size "
                "is accepted for seg_length %d (k = %d)", L, S, stage, L, k);
  return fail(nullptr, MM_EINVAL, "seg_length %d / sketch_size %d exceed the shared-memory budget of %s; the largest sketch "
              "size accepted for seg_length %d (k = %d) is %d", L, S, stage, L, k, lo);
}

int mm_ctx_create(int device, const mm_params *params, mm_ctx **out)
{
  if (!params || !out) return fail(nullptr, MM_EINVAL, "null argument");
  *out = nullptr;
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return fail(nullptr, MM_ENODEVICE, "no CUDA device: %s (this library has no CPU path)", cudaGetErrorString(e));
  if (device < 0 || device >= n_dev) return fail(nullptr, MM_ENODEVICE, "device %d out of range (%d devices)", device, n_dev);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MM_ENODEVICE, "cannot query device");
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, MM_ENODEVICE, "device %d is sm_%d%d; this build is sm_90a only", device, prop.major, prop.minor);
  if (int rc = mm_params_check(params)) return rc;
  mm_ctx *c = new mm_ctx();
  c->device = device;
  c->params = *params;
  c->sm_count = prop.multiProcessorCount;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete c;
    return fail(nullptr, MM_ECUDA, "cannot create stream");
  }
  for (auto &ev : c->ev) cudaEventCreate(&ev);
  cudaEventCreate(&c->ev_pack);
  if (cudaHostAlloc((void **)&c->h_pub, 256, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
    cudaStreamDestroy(c->stream);
    delete c;
    return fail(nullptr, MM_ENOMEM, "cannot allocate the pinned counter page");
  }
  if (const char *g = getenv("MM_BLOCKING_WAIT")) {
    if (g[0] == '1' && cudaEventCreateWithFlags(&c->ev_wait, cudaEventBlockingSync | cudaEventDisableTiming) == cudaSuccess)
      c->blocking_wait = true;
  }
  if (const char *g = getenv("MM_L2_GENERAL")) c->l2_mode = (g[0] == '1') ? 0 : 1; /* test hook: general kernel only */
  if (const char *g = getenv("MM_SKETCH_TABLE")) c->sk_mode = (g[0] == '1') ? 1 : 0; /* test hook: general sketch kernel only */
  if (const char *g = getenv("MM_L1_CTA")) c->l1_warp = (g[0] == '1') ? 0 : 1; /* test hook: general L1 path only */
  if (params->sketch_size > 1000) c->l2_mode = 0; /* the stream kernel packs its counters in 11 bits */
  *out = c;
  return MM_OK;
}

int mm_ctx_destroy(mm_ctx *c)
{
  if (!c) return MM_OK;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  for (auto &ev : c->ev) cudaEventDestroy(ev);
  if (c->h_pub) cudaFreeHost(c->h_pub);
  if (c->ev_wait) cudaEventDestroy(c->ev_wait);
  cudaStreamDestroy(c->stream);
  delete c;
  return MM_OK;
}

const char *mm_last_error(const mm_ctx *c) { return c ? c->error.c_str() : g_create_error.c_str(); }
int mm_ctx_diag(const mm_ctx *ctx, uint64_t out[8])
{
  if (!ctx || !out) return MM_EINVAL;
  memcpy(out, ctx->diag, sizeof(ctx->diag));
  return MM_OK;
}
int mm_ctx_device(const mm_ctx *c) { return c ? c->device : -1; }
uint64_t mm_kernel_launches(const mm_ctx *c) { return c ? c->launches : 0; }

int mm_index_upload(mm_ctx *c, const mm_minmer *mi, uint64_t n_mi, const uint64_t *keys, const uint64_t *offsets,
                    uint64_t n_keys, const mm_ipoint *points, uint64_t n_points, const uint8_t *key_is_freq,
                    const int32_t *contig_len, const int32_t *contig_name_id, const int32_t *contig_group,
                    int32_t n_contigs)
{
  if (!c) return MM_EINVAL;
  if (n_contigs < 1 || !contig_len) return fail(c, MM_EINVAL, "no contigs");
  if (n_keys && (!keys || !offsets || !key_is_freq)) return fail(c, MM_EINVAL, "null lookup arrays");
  if (n_keys && offsets[n_keys] != n_points) return fail(c, MM_EINVAL, "offsets[n_keys] != n_points");
  CU(c, cudaSetDevice(c->device));
  drop_index(c);
  image_guard guard{c};

  /* contig_start: first index entry of each contig; the index must be ordered by (seqId, wpos) */
  std::vector<uint64_t> cstart((size_t)n_contigs + 1, 0);
  {
    int32_t prev_seq = 0, prev_pos = -0x7fffffff;
    for (uint64_t i = 0; i < n_mi; i++) {
      const int32_t s = mi[i].seqId;
      if (s < 0 || s >= n_contigs) return fail(c, MM_EINVAL, "minmer %llu: seqId %d out of range", (unsigned long long)i, s);
      if (s < prev_seq || (s == prev_seq && mi[i].wpos < prev_pos))
        return fail(c, MM_EINVAL, "minmer index not sorted by (seqId, wpos) at entry %llu", (unsigned long long)i);
      if (s != prev_seq) prev_pos = -0x7fffffff;
      prev_seq = s; prev_pos = mi[i].wpos;
      cstart[(size_t)s + 1]++;
    }
    for (int32_t s = 0; s < n_contigs; s++) cstart[(size_t)s + 1] += cstart[(size_t)s];
  }
  int rc = begin_image(c, n_mi, n_keys, n_points, n_contigs);
  if (rc) return rc;
  const mm_blob_header &h = c->hdr;
  mm_devbuf<uint32_t> d_err;
  CU(c, d_err.reserve(1));
  CU(c, cudaMemsetAsync(d_err.get(), 0, 4, c->stream));

  /* AoS records go up in chunks and are re-laid out on the device (SoA index, packed points) */
  {
    const uint64_t CH = 1ULL << 24;
    mm_devbuf<unsigned char> stage;
    CU(c, stage.reserve(CH * 24));
    for (uint64_t at = 0; at < n_mi; at += CH) {
      const uint64_t n = std::min(CH, n_mi - at);
      CU(c, cudaMemcpyAsync(stage.get(), mi + at, n * sizeof(mm_minmer), cudaMemcpyHostToDevice, c->stream));
      CU(c, mm_upload_split_minmers((const mm_minmer *)stage.get(), n, (uint64_t *)(c->blob + h.off_idx_hash) + at,
                                    (int32_t *)(c->blob + h.off_idx_wpos) + at, (int32_t *)(c->blob + h.off_idx_wend) + at,
                                    (int8_t *)(c->blob + h.off_idx_strand) + at, c->stream));
      CU(c, cudaStreamSynchronize(c->stream));
    }
    for (uint64_t at = 0; at < n_points; at += CH) {
      const uint64_t n = std::min(CH, n_points - at);
      CU(c, cudaMemcpyAsync(stage.get(), points + at, n * sizeof(mm_ipoint), cudaMemcpyHostToDevice, c->stream));
      CU(c, mm_upload_pack_points((const mm_ipoint *)stage.get(), n, n_contigs, (uint64_t *)(c->blob + h.off_pts) + at,
                                  d_err.get(), c->stream));
      CU(c, cudaStreamSynchronize(c->stream));
    }
  }
  mm_devbuf<uint64_t> d_keys, d_offs;
  mm_devbuf<uint8_t> d_freq;
  if (n_keys) {
    CU(c, d_keys.reserve(n_keys));
    CU(c, d_offs.reserve(n_keys + 1));
    CU(c, d_freq.reserve(n_keys));
    CU(c, cudaMemcpyAsync(d_keys.get(), keys, n_keys * 8, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(d_offs.get(), offsets, (n_keys + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(d_freq.get(), key_is_freq, n_keys, cudaMemcpyHostToDevice, c->stream));
  }
  return finish_image(c, cstart, d_keys.get(), d_offs.get(), d_freq.get(), d_err.get(), contig_len, contig_name_id, contig_group);
}

int mm_tables_upload(mm_ctx *c, const int32_t *cut, int32_t n_cut, const int32_t *mh, int32_t n_mh)
{
  if (!c || !cut || !mh || n_cut < 1 || n_mh < 1) return fail(c, MM_EINVAL, "bad tables");
  c->cutoffs.assign(cut, cut + n_cut);
  c->min_hits.assign(mh, mh + n_mh);
  CU(c, cudaSetDevice(c->device));
  return write_tables(c);
}

int mm_index_blob(mm_ctx *c, void **blob, uint64_t *n_bytes)
{
  if (!c || !blob || !n_bytes) return MM_EINVAL;
  if (!c->blob_ready) return fail(c, MM_ESTATE, "no index");
  *blob = c->blob; *n_bytes = c->blob_bytes;
  return MM_OK;
}

int mm_index_blob_alloc(mm_ctx *c, uint64_t n_bytes, void **blob)
{
  if (!c || !blob || n_bytes < sizeof(mm_blob_header)) return MM_EINVAL;
  CU(c, cudaSetDevice(c->device));
  drop_index(c);
  CU(c, c->own_blob.reserve(n_bytes));
  c->blob = c->own_blob.get(); c->blob_bytes = n_bytes;
  *blob = c->blob;
  return MM_OK;
}

int mm_index_adopt_blob(mm_ctx *c)
{
  if (!c || !c->blob) return fail(c, MM_ESTATE, "no blob allocated");
  CU(c, cudaSetDevice(c->device));
  CU(c, cudaMemcpyAsync(&c->hdr, c->blob, sizeof(c->hdr), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  if (c->hdr.magic != MM_BLOB_MAGIC || c->hdr.total_bytes != c->blob_bytes) return fail(c, MM_EINVAL, "blob header mismatch");
  resolve_index(c);
  c->blob_ready = true;
  return MM_OK;
}

int mm_ctx_share_index(mm_ctx *c, const mm_ctx *src)
{
  if (!c || !src) return MM_EINVAL;
  if (!src->blob_ready) return fail(c, MM_ESTATE, "source context has no index");
  if (c->device != src->device) return fail(c, MM_EINVAL, "contexts are on different devices");
  cudaSetDevice(c->device);
  drop_index(c);
  c->blob = src->blob; c->blob_bytes = src->blob_bytes;
  c->hdr = src->hdr;
  c->cutoffs = src->cutoffs; c->min_hits = src->min_hits;
  c->share_src = src;
  resolve_index(c);
  c->blob_ready = true;
  return MM_OK;
}

static int batch_upload_any(mm_ctx *c, const void *bases, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs, int packed)
{
  if (!c || (!bases && n_bases) || (!segs && n_segs)) return fail(c, MM_EINVAL, "null argument");
  int rc = upload_batch(c, bases, n_bases, segs, n_segs, packed);
  if (rc) return rc;
  CU(c, wait_stream(c));
  cudaEventElapsedTime(&c->stage_ms[3], c->ev[6], c->ev[7]);
  return MM_OK;
}
int mm_batch_upload(mm_ctx *c, const char *bases, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs)
{
  return batch_upload_any(c, bases, n_bases, segs, n_segs, 0);
}
int mm_batch_upload_packed(mm_ctx *c, const uint8_t *nibbles, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs)
{
  return batch_upload_any(c, nibbles, n_bases, segs, n_segs, 1);
}

int mm_map_resident(mm_ctx *c, uint64_t *n_candidates, uint64_t *n_loci)
{
  if (!c) return MM_EINVAL;
  int rc = run_pipeline(c);
  if (rc) return rc;
  if (n_candidates) *n_candidates = c->n_cands;
  if (n_loci) *n_loci = c->n_loci;
  return MM_OK;
}

int mm_batch_fetch(mm_ctx *c, mm_segment_result *seg_results, mm_l1_candidate *cands, uint64_t cand_cap,
                   mm_l2_locus *loci, uint64_t loci_cap)
{
  if (!c || !c->batch_mapped) return fail(c, MM_ESTATE, "no mapped batch");
  if (cand_cap < c->n_cands || loci_cap < c->n_loci) return fail(c, MM_ECAPACITY, "output capacity too small");
  CU(c, cudaSetDevice(c->device));
  CU(c, cudaEventRecord(c->ev[5], c->stream));
  if (seg_results) CU(c, cudaMemcpyAsync(seg_results, c->d_seg_res.get(), c->n_segs * sizeof(mm_segment_result), cudaMemcpyDeviceToHost, c->stream));
  if (cands && c->n_cands) CU(c, cudaMemcpyAsync(cands, c->d_cands.get(), c->n_cands * sizeof(mm_l1_candidate), cudaMemcpyDeviceToHost, c->stream));
  if (loci && c->n_loci) CU(c, cudaMemcpyAsync(loci, c->d_loci.get(), c->n_loci * sizeof(mm_l2_locus), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaEventRecord(c->ev[6], c->stream));
  CU(c, wait_stream(c));
  cudaEventElapsedTime(&c->stage_ms[4], c->ev[5], c->ev[6]);
  return MM_OK;
}

int mm_batch_fetch_sketch(mm_ctx *c, mm_minmer *out, int32_t *out_count)
{
  if (!c || !c->batch_mapped || !out || !out_count) return fail(c, MM_ESTATE, "no mapped batch");
  CU(c, cudaSetDevice(c->device));
  const uint64_t S = (uint64_t)c->params.sketch_size, n = c->n_segs * S;
  std::vector<uint64_t> hh(n);
  std::vector<int2> pp(n);
  std::vector<int8_t> ss(n);
  std::vector<mm_segment_result> sr(c->n_segs);
  std::vector<mm_segment> sg(c->n_segs);
  CU(c, cudaMemcpyAsync(hh.data(), c->d_sk_hash.get(), n * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(pp.data(), c->d_sk_pos.get(), n * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(ss.data(), c->d_sk_strand.get(), n, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(sr.data(), c->d_seg_res.get(), c->n_segs * sizeof(mm_segment_result), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(sg.data(), c->d_segs.get(), c->n_segs * sizeof(mm_segment), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  for (uint64_t s = 0; s < c->n_segs; s++) {
    out_count[s] = sr[s].sketch_size;
    for (int j = 0; j < sr[s].sketch_size; j++) {
      mm_minmer &m = out[s * S + j];
      m.hash = hh[s * S + j]; m.wpos = pp[s * S + j].x; m.wpos_end = pp[s * S + j].y;
      m.seqId = sg[s].seq_counter; m.strand = ss[s * S + j]; m._pad = 0;
    }
  }
  return MM_OK;
}

int mm_sketch_segments(mm_ctx *c, const char *bases, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs,
                       mm_minmer *out, int32_t *out_count)
{
  if (!c || !out || !out_count || (!segs && n_segs)) return fail(c, MM_EINVAL, "null argument");
  int rc = upload_batch(c, bases, n_bases, segs, n_segs, 0);
  if (rc) return rc;
  if ((rc = launch_pack_if_ascii(c))) return rc;
  ZERO_WORDS(c, c->d_counters.get(), 16);
  CU(c, cudaEventRecord(c->ev[0], c->stream));
  if ((rc = launch_sketch_all(c, false))) return rc; /* sketches only: no index needed */
  CU(c, cudaEventRecord(c->ev[1], c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  cudaEventElapsedTime(&c->stage_ms[0], c->ev[0], c->ev[1]);
  {
    uint32_t h9 = 0;
    if (cudaMemcpy(&h9, c->d_counters.get() + 9, 4, cudaMemcpyDeviceToHost) == cudaSuccess) c->diag[MM_DIAG_SKETCH_GENERAL_SEGMENTS] += h9;
  }
  c->diag[MM_DIAG_LONG_FRAGMENTS] += c->n_long;
  c->batch_mapped = true; /* sketches only; fetch_sketch reads sketch_size == raw count */
  rc = mm_batch_fetch_sketch(c, out, out_count);
  c->batch_mapped = false;
  return rc;
}

static int map_segments_any(mm_ctx *c, const void *bases, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs,
                            mm_segment_result *seg_results, mm_l1_candidate *cands, uint64_t cand_cap, uint64_t *n_candidates,
                            mm_l2_locus *loci, uint64_t loci_cap, uint64_t *n_loci, int packed)
{
  if (!c || !seg_results || !n_candidates || !n_loci) return fail(c, MM_EINVAL, "null argument");
  int rc = upload_batch(c, bases, n_bases, segs, n_segs, packed);
  if (rc) return rc;
  if ((rc = run_pipeline(c))) return rc;
  cudaEventElapsedTime(&c->stage_ms[3], c->ev[6], c->ev[7]);
  *n_candidates = c->n_cands;
  *n_loci = c->n_loci;
  if (cand_cap < c->n_cands || loci_cap < c->n_loci) return fail(c, MM_ECAPACITY, "need %llu candidates, %llu loci", (unsigned long long)c->n_cands, (unsigned long long)c->n_loci);
  return mm_batch_fetch(c, seg_results, cands, cand_cap, loci, loci_cap);
}
int mm_map_segments(mm_ctx *c, const char *bases, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs,
                    mm_segment_result *seg_results, mm_l1_candidate *cands, uint64_t cand_cap, uint64_t *n_candidates,
                    mm_l2_locus *loci, uint64_t loci_cap, uint64_t *n_loci)
{
  return map_segments_any(c, bases, n_bases, segs, n_segs, seg_results, cands, cand_cap, n_candidates, loci, loci_cap, n_loci, 0);
}
int mm_map_segments_packed(mm_ctx *c, const uint8_t *nibbles, uint64_t n_bases, const mm_segment *segs, uint64_t n_segs,
                           mm_segment_result *seg_results, mm_l1_candidate *cands, uint64_t cand_cap, uint64_t *n_candidates,
                           mm_l2_locus *loci, uint64_t loci_cap, uint64_t *n_loci)
{
  return map_segments_any(c, nibbles, n_bases, segs, n_segs, seg_results, cands, cand_cap, n_candidates, loci, loci_cap, n_loci, 1);
}

int mm_ctx_set_wait_mode(mm_ctx *c, int blocking)
{
  if (!c) return MM_EINVAL;
  if (blocking && !c->ev_wait) {
    cudaSetDevice(c->device);
    if (cudaEventCreateWithFlags(&c->ev_wait, cudaEventBlockingSync | cudaEventDisableTiming) != cudaSuccess) {
      c->ev_wait = nullptr;
      return fail(c, MM_ECUDA, "cannot create the blocking event");
    }
  }
  c->blocking_wait = blocking != 0;
  return MM_OK;
}

int mm_ctx_set_phase_hook(mm_ctx *c, mm_phase_hook hook, void *user)
{
  if (!c) return MM_EINVAL;
  c->hook = hook; c->hook_user = user;
  return MM_OK;
}

int mm_last_stage_ms(const mm_ctx *c, float ms[8])
{
  if (!c || !ms) return MM_EINVAL;
  for (int i = 0; i < 8; i++) ms[i] = c->stage_ms[i];
  return MM_OK;
}
int mm_last_pack_ms(const mm_ctx *c, float *ms)
{
  if (!c || !ms) return MM_EINVAL;
  *ms = c->pack_ms;
  return MM_OK;
}

/* pinned host memory for the caller's batch buffers (H2D/D2H at full PCIe rate) */
int mm_host_alloc(void **ptr, uint64_t bytes)
{
  if (!ptr) return MM_EINVAL;
  return cudaHostAlloc(ptr, bytes, cudaHostAllocPortable) == cudaSuccess ? MM_OK : MM_ENOMEM; /* pinned for every device of the process */
}
int mm_host_free(void *ptr) { return cudaFreeHost(ptr) == cudaSuccess ? MM_OK : MM_ECUDA; }

/* skch::Sketch's build + index + computeFreqHist + dropFreqSeedSet on the device (mm_index_build.cu) */
int mm_index_build(mm_ctx *c, const char *seqs, int seqs_on_device, const uint64_t *contig_offsets, int32_t n_contigs,
                   const int32_t *contig_name_id, const int32_t *contig_group, float kmer_pct_threshold, int keep_lookup,
                   mm_index_stats *stats)
{
  if (!c) return MM_EINVAL;
  if (n_contigs < 1 || !contig_offsets || !seqs) return fail(c, MM_EINVAL, "no contigs");
  CU(c, cudaSetDevice(c->device));
  const auto t0 = std::chrono::steady_clock::now();
  drop_index(c);
  image_guard guard{c};
  c->built = mm_built_index{};
  c->built_kept = false;
  const uint64_t total = contig_offsets[n_contigs];
  mm_devbuf<uint8_t> staged;
  if (!seqs_on_device) {
    CU(c, staged.reserve(total + 64));
    CU(c, cudaMemcpyAsync(staged.get(), seqs, total, cudaMemcpyHostToDevice, c->stream));
  }
  mm_built_index B;
  std::string err;
  int rc = mm_build_index_device(c->params, seqs_on_device ? (const uint8_t *)seqs : staged.get(), contig_offsets, n_contigs,
                                 kmer_pct_threshold, c->stream, c->sm_count, &B, err);
  staged.reset();
  if (rc != MM_OK) return fail(c, rc, "index build: %s", err.c_str());
  c->launches += 12;

  const uint64_t n_mi = B.n_minmers, n_keys = B.n_keys, n_points = B.n_points;
  if (n_mi >= (1ULL << 32)) return fail(c, MM_EINVAL, "more than 2^32 minmers");
  /* contig_start from the seqId column */
  std::vector<uint64_t> cstart((size_t)n_contigs + 1, 0);
  if (n_mi) {
    mm_devbuf<unsigned long long> d_cnt;
    CU(c, d_cnt.reserve((size_t)n_contigs + 1));
    CU(c, cudaMemsetAsync(d_cnt.get(), 0, ((size_t)n_contigs + 1) * 8, c->stream));
    CU(c, mm_index_count_seq(n_mi, B.seq.get(), d_cnt.get(), c->stream));
    std::vector<unsigned long long> cnt((size_t)n_contigs + 1);
    CU(c, cudaMemcpyAsync(cnt.data(), d_cnt.get(), ((size_t)n_contigs + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    for (int32_t q = 0; q < n_contigs; q++) cstart[(size_t)q + 1] = cstart[(size_t)q] + cnt[(size_t)q];
  }
  if ((rc = begin_image(c, n_mi, n_keys, n_points, n_contigs))) return rc;
  const mm_blob_header &h = c->hdr;
  if (n_mi) {
    CU(c, cudaMemcpyAsync(c->blob + h.off_idx_hash, B.hash.get(), n_mi * 8, cudaMemcpyDeviceToDevice, c->stream));
    CU(c, cudaMemcpyAsync(c->blob + h.off_idx_wpos, B.wpos.get(), n_mi * 4, cudaMemcpyDeviceToDevice, c->stream));
    CU(c, cudaMemcpyAsync(c->blob + h.off_idx_wend, B.wend.get(), n_mi * 4, cudaMemcpyDeviceToDevice, c->stream));
    CU(c, cudaMemcpyAsync(c->blob + h.off_idx_strand, B.strand.get(), n_mi, cudaMemcpyDeviceToDevice, c->stream));
  }
  if (n_points) CU(c, cudaMemcpyAsync(c->blob + h.off_pts, B.pts.get(), n_points * 8, cudaMemcpyDeviceToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  B.hash.reset(); B.wpos.reset(); B.wend.reset(); B.seq.reset(); B.strand.reset(); /* before the death order's sort */
  mm_devbuf<uint32_t> d_err;
  CU(c, d_err.reserve(1));
  CU(c, cudaMemsetAsync(d_err.get(), 0, 4, c->stream));
  std::vector<int32_t> clen((size_t)n_contigs);
  for (int32_t q = 0; q < n_contigs; q++) clen[(size_t)q] = (int32_t)(contig_offsets[q + 1] - contig_offsets[q]);
  rc = finish_image(c, cstart, B.keys.get(), B.offs.get(), B.is_freq.get(), d_err.get(), clen.data(), contig_name_id, contig_group);
  if (!c->blob_ready) return rc; /* else rc is write_tables': the index stands either way */
  if (stats) {
    memset(stats, 0, sizeof *stats);
    stats->n_minmers = n_mi; stats->n_minmers_before_filter = B.n_minmers_before_filter; stats->n_keys = n_keys; stats->n_points = n_points;
    stats->freq_threshold = B.freq_threshold; stats->n_chunks = B.n_chunks; stats->n_fixed_chunks = B.n_fixed_chunks; stats->fix_rounds = B.fix_rounds;
    stats->hist_min_count = B.hist_min_count; stats->hist_max_count = B.hist_max_count; stats->hist_min_keys = B.hist_min_keys;
    stats->hist_max_keys = B.hist_max_keys; stats->ms_scan = B.ms_scan; stats->ms_post = B.ms_post; stats->ms_lookup = B.ms_lookup;
    stats->ms_total = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  if (keep_lookup) { c->built = std::move(B); c->built_kept = true; }
  return rc;
}

/* host copies of what mm_index_build left on the device (needs keep_lookup); any output may be NULL */
int mm_index_download(mm_ctx *c, mm_minmer *mi, uint64_t *keys, uint64_t *offsets, mm_ipoint *points, uint8_t *is_freq)
{
  if (!c || !c->blob_ready) return fail(c, MM_ESTATE, "no index");
  if ((keys || offsets || points || is_freq) && !c->built_kept) return fail(c, MM_ESTATE, "the lookup arrays were not kept (keep_lookup)");
  CU(c, cudaSetDevice(c->device));
  const mm_blob_header &h = c->hdr;
  if (mi && h.n_minmers) {
    const uint64_t n = h.n_minmers;
    std::vector<uint64_t> hh(n), cs((size_t)h.n_contigs + 1);
    std::vector<int32_t> a(n), b(n);
    std::vector<int8_t> st(n);
    CU(c, cudaMemcpy(hh.data(), c->blob + h.off_idx_hash, n * 8, cudaMemcpyDeviceToHost));
    CU(c, cudaMemcpy(a.data(), c->blob + h.off_idx_wpos, n * 4, cudaMemcpyDeviceToHost));
    CU(c, cudaMemcpy(b.data(), c->blob + h.off_idx_wend, n * 4, cudaMemcpyDeviceToHost));
    CU(c, cudaMemcpy(st.data(), c->blob + h.off_idx_strand, n, cudaMemcpyDeviceToHost));
    CU(c, cudaMemcpy(cs.data(), c->blob + h.off_contig_start, cs.size() * 8, cudaMemcpyDeviceToHost));
    int32_t q = 0;
    for (uint64_t i = 0; i < n; i++) {
      while (i >= cs[(size_t)q + 1]) q++;
      mi[i].hash = hh[i]; mi[i].wpos = a[i]; mi[i].wpos_end = b[i]; mi[i].seqId = q; mi[i].strand = st[i]; mi[i]._pad = 0;
    }
  }
  const mm_built_index &B = c->built;
  if (keys && B.n_keys) CU(c, cudaMemcpy(keys, B.keys.get(), B.n_keys * 8, cudaMemcpyDeviceToHost));
  if (offsets) CU(c, cudaMemcpy(offsets, B.offs.get(), (B.n_keys + 1) * 8, cudaMemcpyDeviceToHost));
  if (is_freq && B.n_keys) CU(c, cudaMemcpy(is_freq, B.is_freq.get(), B.n_keys, cudaMemcpyDeviceToHost));
  if (points && B.n_points) {
    mm_devbuf<mm_ipoint> d;
    CU(c, d.reserve(B.n_points));
    CU(c, mm_index_unpack_points(B.n_points, (const uint64_t *)(c->blob + h.off_pts), B.keys.get(), B.offs.get(), B.n_keys, d.get(),
                                 c->stream));
    CU(c, cudaMemcpyAsync(points, d.get(), B.n_points * sizeof(mm_ipoint), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
  }
  return MM_OK;
}

} // extern "C"
