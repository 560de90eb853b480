/*
 * mm_index_build.cu -- the reference index built on the GPU (SURVEY 8(f)-1).
 *
 * Replaces, for a reference that is already in device memory as text:
 *   CommonFunc::addMinmers        reference src/map/include/commonFunc.hpp:301-570   (sliding-window minmer intervals)
 *   Sketch::index                 winSketch.hpp:379-404                              (hash -> interval points, fusion rule)
 *   Sketch::computeFreqHist / computeFreqSeedSet / dropFreqSeedSet   :410-453, :488-504 (frequent-seed filter)
 * and leaves the device arrays that mm_index_upload would have produced from host arrays.
 *
 * The window scan of addMinmers is a sequential state machine whose every record boundary is an L2 evaluation point, so it
 * is not re-derived: mm_winmachine.h restates it once (tested record for record against the reference on the CPU) and
 * this file runs that machine in parallel over CHUNKS of every contig, one GPU thread per chunk:
 *   k_window_scan   chunk [a, b) starts WARM positions early from an empty machine (records suppressed until a). At a it
 *                   takes a digest of its state, marks the records that are open as "started earlier", scans to b, takes
 *                   another digest and exports which hashes are open (with the start of their record).
 *   host            chunk j is accepted iff chunk j-1 is, digest_start(j) == digest_end(j-1) and the machine never took an
 *                   expired heap entry (wm_machine::drained: the only way history older than the window can matter).
 *   k_window_fix    rejected chunks (N runs, low complexity; none on ordinary sequence) are re-scanned by ONE thread per
 *                   run of them that first rebuilds the exact state at the run's start from the accepted chunk before it.
 *   k_patch_starts  a record that was open at its chunk's start gets its wpos from the previous chunk's export.
 * Then the post-processing of :522-568 with scans and radix sorts (malformed records, strand collapse, chunking to <= w,
 * order by (seqId, wpos, wpos_end) -- STABLE in emission order where the reference's std::sort leaves exact ties in
 * libstdc++'s order, see DESIGN.md --, adjacent de-duplication), Sketch::index as a sort by hash + adjacent-record rule,
 * the frequency histogram on the device and its threshold on the host (a few hundred numbers).
 */
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <type_traits>
#include <vector>

#include "mm_index_build.h"
#include "mm_winmachine.h"

namespace {

struct wb_chunk {
  int32_t contig;
  int32_t a, b;    /* k-mer positions [a, b) */
  int32_t npos;    /* positions of the contig (len - k + 1) */
};
struct wb_chunk_out {
  uint64_t d_start, d_end;
  uint32_t n_rec;
  uint32_t flags;  /* 1 machine failure, 2 record buffer full, 4 expired heap entry taken (history-dependent) */
  uint32_t n_open;
  uint32_t _pad;
};
struct wb_open {
  uint64_t hash;
  int32_t wpos;
  uint32_t inherited; /* the record was already open at the chunk's start: wpos is the warm-up machine's, to be resolved */
};
struct wb_chain {
  uint32_t first, n;     /* rejected chunks [first, first + n) */
  uint64_t out_offset;   /* first record slot of the chain in the fix buffer; chunk q gets fix_cap slots at out_offset + (q - first) * fix_cap */
};

struct wb_slab_layout {
  size_t off_ring, off_heap, off_nodes, off_mem, off_mh, off_mslot, off_sfree, bytes;
  int32_t ring_cap, heap_cap, node_cap, mem_cap;
};
wb_slab_layout slab_layout(int w, int s)
{
  wb_slab_layout L;
  L.ring_cap = wm_ring_cap(w); L.heap_cap = wm_heap_cap(w); L.node_cap = wm_node_cap(w); L.mem_cap = wm_mem_cap(s);
  size_t o = 0;
  L.off_ring = o; o += (size_t)L.ring_cap * sizeof(wm_kmer);
  L.off_heap = o; o += (size_t)L.heap_cap * sizeof(wm_kmer);
  L.off_nodes = o; o += (size_t)L.node_cap * sizeof(wm_node);
  o = (o + 15) & ~(size_t)15;
  L.off_mem = o; o += (size_t)L.mem_cap * sizeof(wm_member);
  L.off_mh = o; o += (size_t)L.mem_cap * 8;
  L.off_mslot = o; o += (size_t)L.mem_cap * 2;
  L.off_sfree = o; o += (size_t)L.mem_cap * 2;
  L.bytes = (o + 255) & ~(size_t)255;
  return L;
}
__device__ __forceinline__ void attach(wm_machine &m, unsigned char *slab, const wb_slab_layout &L)
{
  m.ring = (wm_kmer *)(slab + L.off_ring); m.ring_cap = L.ring_cap;
  m.heap = (wm_kmer *)(slab + L.off_heap); m.heap_cap = L.heap_cap;
  m.nodes = (wm_node *)(slab + L.off_nodes); m.node_cap = L.node_cap;
  m.slots = (wm_member *)(slab + L.off_mem); m.mem_cap = L.mem_cap;
  m.mh = (uint64_t *)(slab + L.off_mh); m.mslot = (uint16_t *)(slab + L.off_mslot); m.sfree = (uint16_t *)(slab + L.off_sfree);
}
__device__ __forceinline__ void export_open(const wm_machine &m, wb_open *ex, wb_chunk_out &o)
{
  o.n_open = (uint32_t)m.mem_n;
  for (int32_t j = 0; j < m.mem_n; j++) { const wm_member &e = wm_at(m, j); ex[j].hash = e.hash; ex[j].wpos = e.wpos; ex[j].inherited = e.inherited; }
}
__device__ __forceinline__ int32_t find_open(const wb_open *ex, uint32_t n, uint64_t h)
{
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (ex[mid].hash < h) lo = mid + 1; else hi = mid;
  }
  return (lo < n && ex[lo].hash == h) ? (int32_t)lo : -1;
}

/* pass 1: every chunk on its own, from a warm-up */
template <int K>
__global__ void __launch_bounds__(128)
k_window_scan(const uint8_t *__restrict__ seq, const uint64_t *__restrict__ contig_off, const wb_chunk *__restrict__ chunks,
              uint32_t n_chunks, int w, int s, int warm, unsigned char *slabs, wb_slab_layout L, wm_record *rec_buf, uint32_t rec_cap,
              wb_chunk_out *outs, wb_open *exports, uint32_t export_stride)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, T = gridDim.x * blockDim.x;
  unsigned char *slab = slabs + (size_t)t * L.bytes;
  for (uint32_t c = t; c < n_chunks; c += T) {
    const wb_chunk ch = chunks[c];
    const uint8_t *base = seq + contig_off[ch.contig];
    wm_machine m;
    attach(m, slab, L);
    m.out = rec_buf + (size_t)c * rec_cap; m.out_cap = rec_cap;
    wm_init(m, K, w, s);
    wm_kmer_bytes<K> win;
    wb_chunk_out o;
    o.d_start = 0; o.flags = 0; o._pad = 0;
    if (ch.a > 0) {
      const int32_t from = ch.a - warm > 0 ? ch.a - warm : 0;
      m.emit_from = ch.a;
      wm_scan<K>(m, win, base, from, ch.a, true);
      o.d_start = wm_digest(m, ch.a - 1 + K - w);
      if (m.drained) o.flags |= 4u;
      m.drained = 0;
      for (int32_t j = 0; j < m.mem_n; j++) wm_at(m, j).inherited = 1; /* their records started before a */
      wm_scan<K>(m, win, base, ch.a, ch.b, false);
    } else {
      wm_scan<K>(m, win, base, 0, ch.b, true);
    }
    if (ch.a > 0 && m.drained) o.flags |= 4u; /* a chunk that starts at 0 is exact whatever its heap did */
    o.d_end = wm_digest(m, ch.b - 1 + K - w);
    export_open(m, exports + (size_t)c * export_stride, o);
    if (ch.b == ch.npos) wm_flush(m, ch.npos);
    if (m.out_n >= m.out_cap) o.flags |= 2u;
    else if (m.fail) o.flags |= 1u;
    o.n_rec = (uint32_t)m.out_n;
    outs[c] = o;
  }
}

/* pass 2: a run of rejected chunks, scanned by one thread from the exact state at the run's start */
template <int K>
__global__ void __launch_bounds__(64)
k_window_fix(const uint8_t *__restrict__ seq, const uint64_t *__restrict__ contig_off, const wb_chunk *__restrict__ chunks,
             const wb_chain *__restrict__ chains, uint32_t n_chains, int w, int s, int warm, unsigned char *slabs, wb_slab_layout L,
             wm_record *fix_buf, uint32_t fix_cap, wb_chunk_out *outs, wb_open *exports, uint32_t export_stride)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_chains) return;
  const wb_chain cn = chains[t];
  unsigned char *slab = slabs + (size_t)t * L.bytes;
  wm_machine m;
  attach(m, slab, L);
  wm_record dummy;
  m.out = &dummy; m.out_cap = 0;
  wm_init(m, K, w, s);
  wm_kmer_bytes<K> win;
  const wb_chunk first = chunks[cn.first];
  const uint8_t *base = seq + contig_off[first.contig];
  bool fresh = true;
  if (first.a > 0) { /* rebuild the exact state at first.a: the accepted chunk before it, silently */
    const wb_chunk pv = chunks[cn.first - 1];
    m.emit_from = 0x7fffffff;
    if (pv.a > 0) {
      const int32_t from = pv.a - warm > 0 ? pv.a - warm : 0;
      wm_scan<K>(m, win, base, from, pv.a, true);
      const wb_open *ex = exports + (size_t)(cn.first - 2) * export_stride;
      const uint32_t nx = outs[cn.first - 2].n_open;
      for (int32_t j = 0; j < m.mem_n; j++) {
        const int32_t at = find_open(ex, nx, m.mh[j]);
        if (at >= 0) wm_at(m, j).wpos = ex[at].wpos;
      }
      wm_scan<K>(m, win, base, pv.a, pv.b, false);
    } else {
      wm_scan<K>(m, win, base, 0, pv.b, true);
    }
    fresh = false;
  }
  m.emit_from = 0;
  for (uint32_t q = cn.first; q < cn.first + cn.n; q++) {
    const wb_chunk ch = chunks[q];
    m.out = fix_buf + cn.out_offset + (size_t)(q - cn.first) * fix_cap; m.out_cap = fix_cap; m.out_n = 0;
    m.fail = 0;
    wm_scan<K>(m, win, base, ch.a, ch.b, fresh);
    fresh = false;
    wb_chunk_out o = outs[q];
    o.flags = 8u; /* fixed: exact by construction */
    o.d_end = wm_digest(m, ch.b - 1 + K - w);
    export_open(m, exports + (size_t)q * export_stride, o);
    if (ch.b == ch.npos) wm_flush(m, ch.npos);
    if (m.out_n >= m.out_cap) o.flags |= 2u;
    else if (m.fail) o.flags |= 1u;
    o.n_rec = (uint32_t)m.out_n;
    outs[q] = o;
  }
}

/* A record can stay open over several chunks: an exported entry that was itself inherited takes its start from the previous
 * chunk's (already resolved) export. Sequential along the chunks of a contig, one block per contig, cheap (s entries per chunk). */
__global__ void k_resolve_exports(const uint32_t *__restrict__ contig_first, const uint32_t *__restrict__ contig_n, uint32_t n_used,
                                  const wb_chunk_out *__restrict__ outs, wb_open *exports, uint32_t export_stride, uint32_t *err)
{
  const uint32_t c = blockIdx.x;
  if (c >= n_used) return;
  const uint32_t first = contig_first[c], n = contig_n[c];
  for (uint32_t q = first + 1; q < first + n; q++) {
    const wb_open *pv = exports + (size_t)(q - 1) * export_stride;
    wb_open *cur = exports + (size_t)q * export_stride;
    const uint32_t np = outs[q - 1].n_open;
    for (uint32_t e = threadIdx.x; e < outs[q].n_open; e += blockDim.x) {
      if (!cur[e].inherited) continue;
      const int32_t at = find_open(pv, np, cur[e].hash);
      if (at < 0) { atomicOr(err, 2u); continue; }
      cur[e].wpos = pv[at].wpos;
      cur[e].inherited = 0;
    }
    __syncthreads();
  }
}

/* records of accepted (not re-scanned) chunks that were open at the chunk's start: wpos from the previous chunk's export */
__global__ void k_patch_starts(const wb_chunk *__restrict__ chunks, const wb_chunk_out *__restrict__ outs, uint32_t n_chunks,
                               wm_record *rec_buf, uint32_t rec_cap, const wb_open *__restrict__ exports, uint32_t export_stride,
                               uint32_t *err)
{
  const uint32_t c = blockIdx.x;
  if (c >= n_chunks) return;
  if (chunks[c].a == 0 || (outs[c].flags & 8u)) return;
  const wb_open *ex = exports + (size_t)(c - 1) * export_stride;
  const uint32_t nx = outs[c - 1].n_open;
  wm_record *r = rec_buf + (size_t)c * rec_cap;
  for (uint32_t i = threadIdx.x; i < outs[c].n_rec; i += blockDim.x) {
    if (!r[i].inherited) continue;
    const int32_t at = find_open(ex, nx, r[i].hash);
    if (at < 0) { atomicOr(err, 1u); continue; }
    r[i].wpos = ex[at].wpos;
  }
}

/* ---- post-processing of addMinmers (:522-568) ----------------------------------------------------------------------
 * Record columns come in mm_rec_views. The compiler ignores __restrict__ on struct members but keeps it on locals, so the
 * columns a kernel only reads are named as restricted locals: their loads stay independent of its stores. */

/* chunk buffers -> one raw array in emission order; per record: kept as it is (1) / number of pieces it is cut into */
__global__ void k_gather_raw(const wb_chunk *__restrict__ chunks, const wb_chunk_out *__restrict__ outs, uint32_t n_chunks,
                             const uint64_t *__restrict__ raw_off, const wm_record *__restrict__ rec_buf, uint32_t rec_cap,
                             const wm_record *__restrict__ fix_buf, const uint64_t *__restrict__ fix_off, int w, mm_rec_view raw,
                             uint32_t *keep, uint32_t *pieces)
{
  const uint32_t c = blockIdx.x;
  if (c >= n_chunks) return;
  const wb_chunk_out o = outs[c];
  const wm_record *src = (o.flags & 8u) ? fix_buf + fix_off[c] : rec_buf + (size_t)c * rec_cap;
  const uint64_t at = raw_off[c];
  const int32_t seqId = chunks[c].contig;
  for (uint32_t i = threadIdx.x; i < o.n_rec; i += blockDim.x) {
    const wm_record r = src[i];
    const uint64_t d = at + i;
    raw.hash[d] = r.hash; raw.wpos[d] = r.wpos; raw.wend[d] = r.wpos_end; raw.seq[d] = seqId;
    raw.strand[d] = (int8_t)(r.votes < 0 ? -1 : 1); /* :534 */
    const bool bad = r.wpos < 0 || r.wpos_end < 0 || r.wpos == r.wpos_end; /* :523-528 */
    const int64_t len = (int64_t)r.wpos_end - (int64_t)r.wpos;
    uint32_t k = 0, p = 0;
    if (!bad) {
      if (r.wpos_end > r.wpos + w) p = (uint32_t)ceilf((float)(r.wpos_end - r.wpos) / (float)w); /* :536-537 */
      else k = 1;
      (void)len;
    }
    keep[d] = k; pieces[d] = p;
  }
}
/* kept records first (emission order), then all pieces (parent's emission order, piece index): the vector the reference sorts */
__global__ void k_scatter_records(uint64_t n_raw, mm_rec_view raw, const uint32_t *__restrict__ keep, const uint32_t *__restrict__ pieces,
                                  const uint64_t *__restrict__ keep_off, const uint64_t *__restrict__ piece_off, uint64_t n_keep, int w,
                                  mm_rec_view o)
{
  const uint64_t *__restrict__ r_hash = raw.hash; const int32_t *__restrict__ r_wpos = raw.wpos, *__restrict__ r_wend = raw.wend;
  const int32_t *__restrict__ r_seq = raw.seq; const int8_t *__restrict__ r_strand = raw.strand;
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_raw) return;
  if (keep[i]) {
    const uint64_t d = keep_off[i];
    o.hash[d] = r_hash[i]; o.wpos[d] = r_wpos[i]; o.wend[d] = r_wend[i]; o.seq[d] = r_seq[i]; o.strand[d] = r_strand[i];
  }
  const uint32_t p = pieces[i];
  if (p) {
    const uint64_t d0 = n_keep + piece_off[i];
    const int32_t a = r_wpos[i], e = r_wend[i];
    for (uint32_t c = 0; c < p; c++) { /* :538-553 */
      const uint64_t d = d0 + c;
      o.hash[d] = r_hash[i]; o.seq[d] = r_seq[i]; o.strand[d] = r_strand[i];
      o.wpos[d] = a + (int32_t)c * w;
      const int32_t hi = a + (int32_t)c * w + w;
      o.wend[d] = hi < e ? hi : e;
    }
  }
}
__global__ void k_iota_keys32(uint64_t n, const int32_t *__restrict__ src, uint32_t *keys, uint32_t *vals)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { keys[i] = (uint32_t)src[i]; vals[i] = (uint32_t)i; }
}
__global__ void k_keys_seq_wpos(uint64_t n, const uint32_t *__restrict__ perm, const int32_t *__restrict__ seq, const int32_t *__restrict__ wpos,
                                uint64_t *keys)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const uint32_t j = perm[i]; keys[i] = ((uint64_t)(uint32_t)seq[j] << 32) | (uint64_t)(uint32_t)wpos[j]; }
}
/* gather in sorted order and flag the records std::unique keeps (:563-568: same wpos and hash as the one before, per contig) */
__global__ void k_gather_sorted(uint64_t n, const uint32_t *__restrict__ perm, mm_rec_view in, mm_rec_view o, uint32_t *uniq)
{
  const uint64_t *__restrict__ i_hash = in.hash; const int32_t *__restrict__ i_wpos = in.wpos, *__restrict__ i_wend = in.wend;
  const int32_t *__restrict__ i_seq = in.seq; const int8_t *__restrict__ i_strand = in.strand;
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t j = perm[i];
  o.hash[i] = i_hash[j]; o.wpos[i] = i_wpos[j]; o.wend[i] = i_wend[j]; o.seq[i] = i_seq[j]; o.strand[i] = i_strand[j];
  uint32_t u = 1;
  if (i > 0) {
    const uint32_t p = perm[i - 1];
    if (i_seq[p] == i_seq[j] && i_wpos[p] == i_wpos[j] && i_hash[p] == i_hash[j]) u = 0;
  }
  uniq[i] = u;
}
__global__ void k_compact5(uint64_t n, const uint32_t *__restrict__ flag, const uint64_t *__restrict__ off, mm_rec_view in, mm_rec_view o)
{
  const uint64_t *__restrict__ i_hash = in.hash; const int32_t *__restrict__ i_wpos = in.wpos, *__restrict__ i_wend = in.wend;
  const int32_t *__restrict__ i_seq = in.seq; const int8_t *__restrict__ i_strand = in.strand;
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  const uint64_t d = off[i];
  o.hash[d] = i_hash[i]; o.wpos[d] = i_wpos[i]; o.wend[d] = i_wend[i]; o.seq[d] = i_seq[i]; o.strand[d] = i_strand[i];
}

/* ---- Sketch::index (:379-404) ------------------------------------------------------------------------------------------
 * In hash-sorted order (stable: index order inside a hash) a record opens a new interval unless the previous record of the
 * same hash ends exactly where it starts (then the CLOSE point moves to its end; seqId is not compared, as in the reference). */
__global__ void k_iota_keys64(uint64_t n, const uint64_t *__restrict__ src, uint64_t *keys, uint32_t *vals)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { keys[i] = src[i]; vals[i] = (uint32_t)i; }
}
__global__ void k_lookup_flags(uint64_t n, const uint64_t *__restrict__ hs, const uint32_t *__restrict__ perm, const int32_t *__restrict__ wpos,
                               const int32_t *__restrict__ wend, uint32_t *key_start, uint32_t *run_start)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool ks = i == 0 || hs[i] != hs[i - 1];
  key_start[i] = ks ? 1u : 0u;
  run_start[i] = (ks || wend[perm[i - (i ? 1 : 0)]] != wpos[perm[i]]) ? 1u : 0u;
}
__global__ void k_lookup_emit(uint64_t n, const uint64_t *__restrict__ hs, const uint32_t *__restrict__ perm, const int32_t *__restrict__ wpos,
                              const int32_t *__restrict__ wend, const int32_t *__restrict__ seq, const uint32_t *__restrict__ key_start,
                              const uint32_t *__restrict__ run_start, const uint64_t *__restrict__ key_idx, const uint64_t *__restrict__ run_idx,
                              uint64_t *keys, uint64_t *offs, uint64_t *pts, uint64_t *rec_key)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t j = perm[i];
  /* exclusive scans of the start flags: at a start the index of the new run / key, elsewhere that index + 1 */
  const uint64_t r = run_start[i] ? run_idx[i] : run_idx[i] - 1;
  const uint64_t k = key_start[i] ? key_idx[i] : key_idx[i] - 1;
  rec_key[i] = k;
  if (key_start[i]) { keys[k] = hs[i]; offs[k] = 2 * r; }
  /* the run's OPEN point carries the seqId of its first record, and so does its CLOSE point (only its pos is moved, :397) */
  if (run_start[i]) pts[2 * r] = mm_pack_point(seq[j], wpos[j], 1);
  const bool last_of_run = i + 1 == n || run_start[i + 1];
  if (last_of_run) {
    /* first record of this run: walk back (runs are almost always one or two records long) */
    uint64_t f = i;
    while (!run_start[f]) f--;
    pts[2 * r + 1] = mm_pack_point(seq[perm[f]], wend[j], 0);
  }
}
__global__ void k_key_counts(uint64_t n_keys, const uint64_t *__restrict__ offs, uint64_t n_points, uint32_t *cnt)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_keys) cnt[i] = (uint32_t)((i + 1 < n_keys ? offs[i + 1] : n_points) - offs[i]);
}
__global__ void k_histogram(uint64_t n_keys, const uint32_t *__restrict__ cnt, unsigned long long *hist, uint32_t hist_n)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_keys) atomicAdd(&hist[cnt[i] < hist_n ? cnt[i] : hist_n - 1], 1ULL);
}
__global__ void k_mark_freq(uint64_t n_keys, const uint32_t *__restrict__ cnt, uint32_t threshold, uint8_t *is_freq)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_keys) is_freq[i] = cnt[i] >= threshold ? 1 : 0;
}
/* a shard of a contig-sharded index: the frequent seeds are the listed ones (ascending), not those above a local threshold */
__device__ __forceinline__ bool in_sorted(const uint64_t *__restrict__ a, uint64_t n, uint64_t h)
{
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (a[mid] < h) lo = mid + 1; else hi = mid;
  }
  return lo < n && a[lo] == h;
}
__global__ void k_mark_listed(uint64_t n_keys, const uint64_t *__restrict__ keys, const uint64_t *__restrict__ freq, uint64_t n_freq,
                              uint8_t *is_freq)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_keys) is_freq[i] = in_sorted(freq, n_freq, keys[i]) ? 1 : 0;
}
__global__ void k_flag_absent(uint64_t n_freq, const uint64_t *__restrict__ freq, const uint64_t *__restrict__ keys, uint64_t n_keys,
                              uint32_t *absent)
{
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_freq) absent[j] = in_sorted(keys, n_keys, freq[j]) ? 0u : 1u;
}
/* the listed hashes the shard lacks: frequent keys with no points after its own keys, so that every shard drops them */
__global__ void k_append_absent(uint64_t n_freq, const uint64_t *__restrict__ freq, const uint32_t *__restrict__ absent,
                                const uint64_t *__restrict__ at, uint64_t n_keys, uint64_t n_points, uint64_t *keys, uint64_t *offs,
                                uint8_t *is_freq)
{
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_freq || !absent[j]) return;
  const uint64_t d = n_keys + at[j];
  keys[d] = freq[j]; offs[d] = n_points; is_freq[d] = 1;
}

/* keep[index position] = the record's hash is not a frequent seed (dropFreqSeedSet :497-504) */
__global__ void k_keep_not_freq(uint64_t n, const uint32_t *__restrict__ perm, const uint64_t *__restrict__ rec_key, const uint8_t *__restrict__ is_freq,
                                uint32_t *keep)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep[perm[i]] = is_freq[rec_key[i]] ? 0u : 1u;
}

#define CE(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) { err = std::string(#call) + ": " + cudaGetErrorString(e_); return e_ == cudaErrorMemoryAllocation ? MM_ENOMEM : MM_ECUDA; } \
  } while (0)

inline uint32_t blocks(uint64_t n, uint32_t per = 256) { return (uint32_t)((n + per - 1) / per); }

#define MM_FOR_EACH_K(X) \
  X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16) X(17) X(18) X(19) X(20) X(21) X(22) X(23) X(24) X(25) X(26) X(27) \
  X(28) X(29) X(30) X(31) X(32)

/* f(std::integral_constant<int, K>()) for a k-mer size K that is compiled in (mm_sketch_kmer_supported) */
template <typename F>
void for_kmer(int K, F &&f)
{
  switch (K) {
#define X(KK) case KK: f(std::integral_constant<int, KK>()); break;
    MM_FOR_EACH_K(X)
#undef X
  }
}

/* cub's two-call convention: call(nullptr, bytes) sizes the temporary storage, which is then held in tmp for the real call */
template <typename Call>
cudaError_t cub_run(mm_devbuf<uint8_t> &tmp, Call &&call)
{
  size_t bytes = 0;
  cudaError_t e = call(nullptr, bytes);
  if (e == cudaSuccess) e = tmp.reserve(bytes + 16);
  return e == cudaSuccess ? call(tmp.get(), bytes) : e;
}

/* off[i] = flag[0] + ... + flag[i - 1] (n > 0), and total = the sum of all n flags; `st` is synchronised once */
cudaError_t count_flags(const uint32_t *flag, uint64_t *off, uint64_t n, cudaStream_t st, uint64_t &total)
{
  const cub::TransformInputIterator<uint64_t, cub::CastOp<uint64_t>, const uint32_t *> in(flag, cub::CastOp<uint64_t>());
  mm_devbuf<uint8_t> tmp;
  cudaError_t e = cub_run(tmp, [&](void *t, size_t &bytes) { return cub::DeviceScan::ExclusiveSum(t, bytes, in, off, (int64_t)n, st); });
  uint64_t last_off = 0; uint32_t last_flag = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&last_off, off + n - 1, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&last_flag, flag + n - 1, 4, cudaMemcpyDeviceToHost, st);
  const cudaError_t s = cudaStreamSynchronize(st); /* before the temporary goes and the last values are read */
  total = last_off + last_flag;
  return e != cudaSuccess ? e : s;
}
template <typename KeyT>
cudaError_t sort_pairs(KeyT *k_in, KeyT *k_out, uint32_t *v_in, uint32_t *v_out, uint64_t n, int end_bit, cudaStream_t st)
{
  mm_devbuf<uint8_t> tmp;
  const cudaError_t e = cub_run(tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceRadixSort::SortPairs(t, bytes, k_in, k_out, v_in, v_out, (int64_t)n, 0, end_bit, st);
  });
  const cudaError_t s = cudaStreamSynchronize(st); /* before the temporary goes */
  return e != cudaSuccess ? e : s;
}

struct stage_events { /* the builder's timing events (ms_scan, ms_post and ms_lookup lie between them), destroyed on every return */
  cudaEvent_t e[4] = {};
  ~stage_events() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
  cudaError_t create()
  {
    for (cudaEvent_t &x : e)
      if (const cudaError_t r = cudaEventCreate(&x)) { x = nullptr; return r; }
    return cudaSuccess;
  }
};

/* ---- chunks ---- */
struct chunk_plan {
  std::vector<wb_chunk> chunks; /* contig by contig, in order */
  int chunk_len;
};
int plan_chunks(int K, const uint64_t *h_contig_off, int32_t n_contigs, chunk_plan &plan, std::string &err)
{
  plan.chunk_len = 16384;
  if (const char *e = getenv("MM_INDEX_CHUNK")) plan.chunk_len = std::max(1024, atoi(e)); /* tests: small chunks */
  for (int32_t c = 0; c < n_contigs; c++) {
    const uint64_t len = h_contig_off[c + 1] - h_contig_off[c];
    if (len >= (1ULL << 31)) { err = "a contig is longer than 2^31 bases"; return MM_EINVAL; }
    const int32_t npos = (int32_t)len - K + 1;
    if (npos <= 0) continue;
    for (int32_t a = 0; a < npos; a += plan.chunk_len) plan.chunks.push_back(wb_chunk{c, a, std::min(npos, a + plan.chunk_len), npos});
  }
  return MM_OK;
}

/* ---- acceptance, fix-up rounds ----
 * A chunk is good if it starts a contig and ran clean, or if its predecessor is good, it ran clean (no failure, no
 * expired heap entry taken) and its state digest at its start equals its predecessor's at its end. A chunk that is not
 * good starts a chain of rejected chunks, or joins the chain right before it; a chain starts right after a good chunk
 * and is re-scanned by one thread from that chunk's exact end state.
 * A chunk right after a chain that is not re-scanned yet is decided in a later round, against the chain's exact end
 * state (it is pending, and so is every chunk after it), unless it failed on its own, which rejects it whatever came
 * before it: then it joins the chain at once. A chain whose next chunk does not match its new end state is extended by
 * that chunk and re-scanned as a whole. So each contig has at most one dirty chain per round, and all of the contig
 * before that chain is good: the chain's start state (chunk first-1 and the resolved exports of first-2) depends on
 * nothing that is rewritten in the same round. The export resolution stops at the dirty chain too, since the exports of
 * pending chunks inherit record starts from the chunks the chain is about to rewrite; what it resolved is final, so
 * the next round resolves from there on. A round decides at least the chunk after each chain it re-scanned, so there
 * are at most as many rounds as chunks; a contig with r separate runs of rejected chunks takes about r rounds.
 * chunk_rounds is that bookkeeping, on the host and without CUDA calls: it decides a round from the chunks' outputs as
 * copied back after the scan or the last re-scan, and names the chains to re-scan and the exports to resolve first. */
struct chunk_rounds {
  enum : uint8_t { CH_GOOD, CH_DIRTY, CH_PENDING };
  struct HostChain { uint32_t first, n; bool dirty; };
  std::vector<uint32_t> cf, cnn; /* chunks of each contig (for the sequential resolution of inherited record starts) */
  std::vector<uint8_t> state; std::vector<int32_t> in_chain; std::vector<HostChain> hchains;
  std::vector<uint32_t> resolve_n; /* per contig: the chunks whose exports the next resolution may touch */
  std::vector<uint32_t> resolved; /* per contig: its chunks up to this one have resolved exports */
  std::vector<uint32_t> res_first, res_n; /* the resolution to run: chunks [res_first, res_first + res_n) of each contig */
  uint64_t decided_before = 0;
  uint32_t n_rounds = 0;
  explicit chunk_rounds(const std::vector<wb_chunk> &chunks) : state(chunks.size(), CH_PENDING), in_chain(chunks.size(), -1)
  {
    for (uint32_t c = 0; c < (uint32_t)chunks.size(); c++) {
      if (c == 0 || chunks[c].contig != chunks[c - 1].contig) { cf.push_back(c); cnn.push_back(0); }
      cnn.back()++;
    }
    resolve_n.resize(cf.size()); resolved.assign(cf.size(), 0); res_first.resize(cf.size()); res_n.resize(cf.size());
  }

  /* decides every chunk it can from outs. chains: the dirty chains, re-scanned in this round (none: every chunk is
   * decided); resolve_n: the exports to resolve before they are */
  int next(const std::vector<wb_chunk_out> &outs, std::vector<wb_chain> &chains, std::string &err)
  {
    uint64_t decided = 0;
    for (size_t g = 0; g < cf.size(); g++) {
      resolve_n[g] = cnn[g];
      for (uint32_t c = cf[g]; c < cf[g] + cnn[g]; c++) {
        const bool first = c == cf[g];
        if (in_chain[c] >= 0) { /* re-scanned in an earlier round: exact (a chain is only dirty from the chunk that made it so on) */
          if (outs[c].flags & 3u) { err = "window machine capacity exceeded while re-scanning a chunk"; return MM_ECAPACITY; }
          state[c] = CH_GOOD;
        } else {
          const uint8_t prev = first ? CH_GOOD : state[c - 1];
          const bool own_fail = (outs[c].flags & (first ? 3u : 7u)) != 0;
          if (prev == CH_GOOD && !own_fail && (first || outs[c].d_start == outs[c - 1].d_end)) {
            state[c] = CH_GOOD;
          } else if (prev == CH_PENDING || (prev == CH_DIRTY && !own_fail)) {
            state[c] = CH_PENDING;
          } else {
            if (!first && in_chain[c - 1] >= 0) { /* the chain before it grows by this chunk and is re-scanned as a whole */
              HostChain &hc = hchains[(size_t)in_chain[c - 1]];
              hc.n++; hc.dirty = true;
              in_chain[c] = in_chain[c - 1];
            } else {
              in_chain[c] = (int32_t)hchains.size();
              hchains.push_back(HostChain{c, 1, true});
            }
            state[c] = CH_DIRTY;
            resolve_n[g] = std::min(resolve_n[g], hchains[(size_t)in_chain[c]].first - cf[g]);
          }
        }
        if (state[c] != CH_PENDING) decided++;
      }
    }
    chains.clear();
    for (HostChain &hc : hchains)
      if (hc.dirty) { chains.push_back(wb_chain{hc.first, hc.n, 0}); hc.dirty = false; }
    if (chains.empty()) return MM_OK;
    if (n_rounds > 0 && decided <= decided_before) { err = "chunk stitching made no progress"; return MM_ECUDA; }
    decided_before = decided;
    n_rounds++;
    return MM_OK;
  }

  /* the next resolution: chunks (resolved, limit) of each contig */
  void resolve_upto(const std::vector<uint32_t> &limit)
  {
    for (size_t g = 0; g < cf.size(); g++) {
      res_first[g] = cf[g] + resolved[g];
      res_n[g] = limit[g] > resolved[g] ? limit[g] - resolved[g] : 0;
      if (limit[g] > resolved[g]) resolved[g] = limit[g] - 1;
    }
  }

  bool converged() const { return std::all_of(state.begin(), state.end(), [](uint8_t x) { return x == CH_GOOD; }); }
  uint32_t n_fixed() const { uint32_t n = 0; for (const HostChain &hc : hchains) n += hc.n; return n; }
};

/* the records of every chunk in emission order, and per record: kept as it is (keep) / number of pieces it is cut into */
struct raw_records { mm_rec_cols cols; mm_devbuf<uint32_t> keep, pieces; uint64_t n = 0; };

/* the window scan of every chunk, the re-scan rounds and the record starts; sets out->fix_rounds and out->n_fixed_chunks */
int scan_windows(const mm_params &p, const uint8_t *d_seq, const uint64_t *h_contig_off, int32_t n_contigs, const chunk_plan &plan,
                 cudaStream_t st, int sm_count, raw_records &raw, mm_built_index *out, std::string &err)
{
  const std::vector<wb_chunk> &chunks = plan.chunks;
  const uint32_t n_chunks = (uint32_t)chunks.size();
  if (!n_chunks) return MM_OK;
  const int K = p.kmer_size, w = p.seg_length, s = p.sketch_size, warm = w + 2 * K + 64;
  mm_devbuf<uint64_t> d_off; mm_devbuf<wb_chunk> d_chunks;
  CE(d_off.reserve((uint64_t)n_contigs + 1));
  CE(cudaMemcpyAsync(d_off.get(), h_contig_off, ((size_t)n_contigs + 1) * 8, cudaMemcpyHostToDevice, st));
  CE(d_chunks.reserve(n_chunks));
  CE(cudaMemcpyAsync(d_chunks.get(), chunks.data(), (size_t)n_chunks * sizeof(wb_chunk), cudaMemcpyHostToDevice, st));
  const wb_slab_layout L = slab_layout(w, s);
  int tpsm = 768; /* machines per SM: the scan is latency-bound (dependent accesses to a per-thread slab), more threads hide more */
  if (const char *e = getenv("MM_INDEX_TPSM")) tpsm = std::max(128, atoi(e) / 128 * 128);
  uint32_t threads = (uint32_t)sm_count * (uint32_t)tpsm;
  if (threads > n_chunks) threads = (n_chunks + 127) / 128 * 128;
  const uint32_t rec_cap = (uint32_t)(plan.chunk_len / 4 + s + 64);
  { /* one slab per machine (~0.4 MB at -s 5000): at 3 Gbp the slabs of a full grid and the chunks' record buffers
     * together exceed an 80 GB device next to the caller's data, so the grid shrinks to the memory that is free
     * (a smaller grid only scans more chunks per thread) */
    size_t free_b = 0, total_b = 0;
    CE(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t fixed = (uint64_t)n_chunks * rec_cap * sizeof(wm_record) + (uint64_t)n_chunks * wm_mem_cap(s) * sizeof(wb_open) + (1ULL << 30);
    const uint64_t room = free_b > fixed ? (free_b - fixed) / 10 * 8 : 0;
    const uint64_t fit = room / L.bytes / 128 * 128;
    if (fit < threads) threads = (uint32_t)std::max<uint64_t>(fit, 128);
  }
  if (const char *e = getenv("MM_INDEX_MACHINES")) { /* tests: a small grid, so that each machine scans many chunks */
    const uint32_t cap = (uint32_t)std::max<long>(128, (strtol(e, nullptr, 10) + 127) / 128 * 128);
    threads = std::min(threads, cap);
  }
  const uint32_t grid = threads / 128;
  const uint32_t stride = (uint32_t)wm_mem_cap(s);
  mm_devbuf<unsigned char> slabs; mm_devbuf<wm_record> rec; mm_devbuf<wb_chunk_out> d_outs; mm_devbuf<wb_open> d_ex;
  CE(slabs.reserve((uint64_t)threads * L.bytes)); CE(rec.reserve((uint64_t)n_chunks * rec_cap));
  CE(d_outs.reserve(n_chunks)); CE(d_ex.reserve((uint64_t)n_chunks * stride));
  for_kmer(K, [&](auto k) {
    k_window_scan<decltype(k)::value><<<grid, 128, 0, st>>>(d_seq, d_off.get(), d_chunks.get(), n_chunks, w, s, warm, slabs.get(), L, rec.get(),
                                                            rec_cap, d_outs.get(), d_ex.get(), stride);
  });
  CE(cudaGetLastError());
  std::vector<wb_chunk_out> outs(n_chunks);
  CE(cudaMemcpyAsync(outs.data(), d_outs.get(), (size_t)n_chunks * sizeof(wb_chunk_out), cudaMemcpyDeviceToHost, st));
  CE(cudaStreamSynchronize(st));

  chunk_rounds rounds(chunks);
  const uint32_t n_used = (uint32_t)rounds.cf.size();
  mm_devbuf<uint32_t> d_cf, d_cn, d_err;
  CE(d_cf.reserve(n_used)); CE(d_cn.reserve(n_used)); CE(d_err.reserve(1));
  CE(cudaMemsetAsync(d_err.get(), 0, 4, st));
  auto resolve = [&](const std::vector<uint32_t> &limit) { /* resolve chunks (resolved, limit) of each contig */
    rounds.resolve_upto(limit);
    cudaError_t e = cudaMemcpyAsync(d_cf.get(), rounds.res_first.data(), (size_t)n_used * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_cn.get(), rounds.res_n.data(), (size_t)n_used * 4, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    k_resolve_exports<<<n_used, 128, 0, st>>>(d_cf.get(), d_cn.get(), n_used, d_outs.get(), d_ex.get(), stride, d_err.get());
    return cudaGetLastError();
  };
  mm_devbuf<wm_record> fix;
  std::vector<uint64_t> fix_off(n_chunks, 0);
  uint64_t fix_used = 0;
  const uint32_t fix_cap = (uint32_t)(3 * plan.chunk_len + s + 64); /* at most three records per position */
  for (;;) {
    std::vector<wb_chain> chains;
    const int rc = rounds.next(outs, chains, err);
    if (rc != MM_OK) return rc;
    if (chains.empty()) break;
    out->fix_rounds = rounds.n_rounds;
    uint64_t need = 0;
    for (auto &cn : chains) { cn.out_offset = fix_used + need; need += (uint64_t)cn.n * fix_cap; }
    if ((fix_used + need) * sizeof(wm_record) > (48ULL << 30)) { err = "too many chunks need an exact re-scan (N-rich / low-complexity reference): use the host builder"; return MM_ECAPACITY; }
    if (fix_used + need > fix.capacity()) /* grow, keeping what earlier rounds wrote */
      CE(fix.reserve_keep((fix_used + need) + (fix_used + need) / 2, fix_used, st));
    for (auto &cn : chains)
      for (uint32_t q = 0; q < cn.n; q++) fix_off[cn.first + q] = cn.out_offset + (uint64_t)q * fix_cap;
    fix_used += need;
    CE(resolve(rounds.resolve_n)); /* the re-scan takes record starts from the exports of the chunks before the chain */
    const uint32_t n_chains = (uint32_t)chains.size();
    mm_devbuf<wb_chain> d_chains;
    CE(d_chains.reserve(n_chains));
    CE(cudaMemcpyAsync(d_chains.get(), chains.data(), n_chains * sizeof(wb_chain), cudaMemcpyHostToDevice, st));
    mm_devbuf<unsigned char> chain_slabs; /* more chains than machines */
    if (n_chains > threads) CE(chain_slabs.reserve((uint64_t)n_chains * L.bytes));
    unsigned char *fslabs = chain_slabs ? chain_slabs.get() : slabs.get();
    for_kmer(K, [&](auto k) {
      k_window_fix<decltype(k)::value><<<(n_chains + 63) / 64, 64, 0, st>>>(d_seq, d_off.get(), d_chunks.get(), d_chains.get(), n_chains, w, s,
                                                                            warm, fslabs, L, fix.get(), fix_cap, d_outs.get(), d_ex.get(), stride);
    });
    CE(cudaGetLastError());
    CE(cudaMemcpyAsync(outs.data(), d_outs.get(), (size_t)n_chunks * sizeof(wb_chunk_out), cudaMemcpyDeviceToHost, st));
    CE(cudaStreamSynchronize(st));
  }
  out->n_fixed_chunks = rounds.n_fixed();
  if (!rounds.converged()) { err = "chunk stitching did not converge"; return MM_ECUDA; }
  slabs.reset();

  CE(resolve(rounds.cnn));
  k_patch_starts<<<n_chunks, 128, 0, st>>>(d_chunks.get(), d_outs.get(), n_chunks, rec.get(), rec_cap, d_ex.get(), stride, d_err.get());
  CE(cudaGetLastError());
  uint32_t h_err = 0;
  CE(cudaMemcpyAsync(&h_err, d_err.get(), 4, cudaMemcpyDeviceToHost, st));
  CE(cudaStreamSynchronize(st));
  if (h_err) { err = "a record open at a chunk start is missing from the previous chunk's export (code " + std::to_string(h_err) + ")"; return MM_ECUDA; }
  d_ex.reset();

  /* ---- raw records in emission order ---- */
  std::vector<uint64_t> raw_off(n_chunks + 1, 0);
  for (uint32_t c = 0; c < n_chunks; c++) raw_off[c + 1] = raw_off[c] + outs[c].n_rec;
  raw.n = raw_off[n_chunks];
  mm_devbuf<uint64_t> d_raw_off, d_fix_off;
  CE(d_raw_off.reserve((uint64_t)n_chunks + 1)); CE(d_fix_off.reserve(n_chunks));
  CE(cudaMemcpyAsync(d_raw_off.get(), raw_off.data(), ((size_t)n_chunks + 1) * 8, cudaMemcpyHostToDevice, st));
  CE(cudaMemcpyAsync(d_fix_off.get(), fix_off.data(), (size_t)n_chunks * 8, cudaMemcpyHostToDevice, st));
  CE(raw.cols.reserve(raw.n)); CE(raw.keep.reserve(raw.n)); CE(raw.pieces.reserve(raw.n));
  k_gather_raw<<<n_chunks, 256, 0, st>>>(d_chunks.get(), d_outs.get(), n_chunks, d_raw_off.get(), rec.get(), rec_cap, fix.get(), d_fix_off.get(),
                                         w, raw.cols.view(), raw.keep.get(), raw.pieces.get());
  CE(cudaGetLastError());
  CE(cudaStreamSynchronize(st));
  return MM_OK;
}

/* kept records + pieces -> the vector the reference sorts, ordered by (seqId, wpos, wpos_end) and de-duplicated: m[n_mi].
 * raw is freed once it is expanded */
int expand_and_sort(raw_records &raw, int32_t n_contigs, int w, cudaStream_t st, mm_rec_cols &m, uint64_t &n_mi, std::string &err)
{
  n_mi = 0;
  if (!raw.n) return MM_OK;
  const uint64_t n_raw = raw.n;
  mm_rec_cols a; /* kept records, then pieces */
  uint64_t n_all = 0;
  {
    mm_devbuf<uint64_t> keep_off, piece_off;
    CE(keep_off.reserve(n_raw + 1)); CE(piece_off.reserve(n_raw + 1));
    uint64_t n_keep = 0, n_pieces = 0;
    CE(count_flags(raw.keep.get(), keep_off.get(), n_raw, st, n_keep));
    CE(count_flags(raw.pieces.get(), piece_off.get(), n_raw, st, n_pieces));
    n_all = n_keep + n_pieces;
    if (n_all >= (1ULL << 32)) { err = "more than 2^32 minmer records"; return MM_EINVAL; }
    CE(a.reserve(n_all));
    k_scatter_records<<<blocks(n_raw), 256, 0, st>>>(n_raw, raw.cols.view(), raw.keep.get(), raw.pieces.get(), keep_off.get(), piece_off.get(),
                                                     n_keep, w, a.view());
    CE(cudaGetLastError());
    CE(cudaStreamSynchronize(st));
  }
  raw.cols.reset(); raw.keep.reset(); raw.pieces.reset();
  if (!n_all) return MM_OK;

  /* ---- order by (seqId, wpos, wpos_end), stable; adjacent de-duplication ---- */
  mm_devbuf<uint32_t> va, vb;
  {
    mm_devbuf<uint32_t> k32a, k32b;
    CE(k32a.reserve(n_all)); CE(k32b.reserve(n_all)); CE(va.reserve(n_all)); CE(vb.reserve(n_all));
    k_iota_keys32<<<blocks(n_all), 256, 0, st>>>(n_all, a.wend.get(), k32a.get(), va.get());
    CE(sort_pairs<uint32_t>(k32a.get(), k32b.get(), va.get(), vb.get(), n_all, 32, st));   /* by wpos_end */
  }
  {
    mm_devbuf<uint64_t> k64a, k64b;
    CE(k64a.reserve(n_all)); CE(k64b.reserve(n_all));
    k_keys_seq_wpos<<<blocks(n_all), 256, 0, st>>>(n_all, vb.get(), a.seq.get(), a.wpos.get(), k64a.get());
    int end_bit = 32;
    while ((1LL << (end_bit - 32)) < (long long)n_contigs + 1) end_bit++;
    CE(sort_pairs<uint64_t>(k64a.get(), k64b.get(), vb.get(), va.get(), n_all, end_bit, st)); /* then by (seqId, wpos): LSD, stable */
  }
  vb.reset();
  mm_rec_cols s; mm_devbuf<uint32_t> uniq;
  CE(s.reserve(n_all)); CE(uniq.reserve(n_all));
  k_gather_sorted<<<blocks(n_all), 256, 0, st>>>(n_all, va.get(), a.view(), s.view(), uniq.get());
  CE(cudaGetLastError());
  CE(cudaStreamSynchronize(st));
  va.reset(); a.reset();
  mm_devbuf<uint64_t> uoff;
  CE(uoff.reserve(n_all + 1));
  CE(count_flags(uniq.get(), uoff.get(), n_all, st, n_mi));
  CE(m.reserve(n_mi));
  k_compact5<<<blocks(n_all), 256, 0, st>>>(n_all, uniq.get(), uoff.get(), s.view(), m.view());
  CE(cudaGetLastError());
  CE(cudaStreamSynchronize(st));
  return MM_OK;
}

/* Sketch::index over m[n_mi] (n_mi > 0): out's keys, offsets, points and every key's count; for the frequency filter, the
 * index position of each record in hash order (perm) and its key (rec_key) */
int index_lookup(const mm_rec_cols &m, uint64_t n_mi, cudaStream_t st, mm_devbuf<uint32_t> &perm, mm_devbuf<uint64_t> &rec_key,
                 mm_built_index *out, std::string &err)
{
  mm_devbuf<uint64_t> hs;
  {
    mm_devbuf<uint64_t> hk; mm_devbuf<uint32_t> va;
    CE(hk.reserve(n_mi)); CE(hs.reserve(n_mi)); CE(va.reserve(n_mi)); CE(perm.reserve(n_mi));
    k_iota_keys64<<<blocks(n_mi), 256, 0, st>>>(n_mi, m.hash.get(), hk.get(), va.get());
    CE(sort_pairs<uint64_t>(hk.get(), hs.get(), va.get(), perm.get(), n_mi, 64, st));
  }
  {
    mm_devbuf<uint32_t> key_start, run_start; mm_devbuf<uint64_t> key_idx, run_idx;
    CE(key_start.reserve(n_mi)); CE(run_start.reserve(n_mi)); CE(key_idx.reserve(n_mi + 1)); CE(run_idx.reserve(n_mi + 1));
    CE(rec_key.reserve(n_mi));
    k_lookup_flags<<<blocks(n_mi), 256, 0, st>>>(n_mi, hs.get(), perm.get(), m.wpos.get(), m.wend.get(), key_start.get(), run_start.get());
    uint64_t n_runs = 0;
    CE(count_flags(key_start.get(), key_idx.get(), n_mi, st, out->n_keys));
    CE(count_flags(run_start.get(), run_idx.get(), n_mi, st, n_runs));
    out->n_points = 2 * n_runs;
    /* exclusive scans give, at a start flag, the index of the new key / run; at other records index + 1 of the current one */
    CE(out->keys.reserve(out->n_keys)); CE(out->offs.reserve(out->n_keys + 1)); CE(out->pts.reserve(out->n_points + 1));
    CE(out->is_freq.reserve(out->n_keys));
    k_lookup_emit<<<blocks(n_mi), 256, 0, st>>>(n_mi, hs.get(), perm.get(), m.wpos.get(), m.wend.get(), m.seq.get(), key_start.get(),
                                                run_start.get(), key_idx.get(), run_idx.get(), out->keys.get(), out->offs.get(), out->pts.get(),
                                                rec_key.get());
    CE(cudaGetLastError());
    CE(cudaMemcpyAsync(out->offs.get() + out->n_keys, &out->n_points, 8, cudaMemcpyHostToDevice, st));
    CE(cudaStreamSynchronize(st));
  }
  hs.reset();
  /* histogram of interval points per key (winSketch.hpp:415-417) */
  CE(out->counts.reserve(out->n_keys));
  k_key_counts<<<blocks(out->n_keys), 256, 0, st>>>(out->n_keys, out->offs.get(), out->n_points, out->counts.get());
  return MM_OK;
}

/* the frequent keys by `rule` (computeFreqHist, or the listed hashes) flagged in out->is_freq, then dropFreqSeedSet: the
 * records of m[n_mi] with the other hashes, in out->mi. perm and rec_key are freed once used */
int frequency_filter(const mm_freq_rule &rule, const mm_rec_cols &m, uint64_t n_mi, mm_devbuf<uint32_t> &perm, mm_devbuf<uint64_t> &rec_key,
                     cudaStream_t st, mm_built_index *out, std::string &err)
{
  const uint64_t n_keys = out->n_keys;
  uint32_t *cnt = out->counts.get();
  if (rule.mode == mm_freq_rule::OWN_THRESHOLD) { /* the frequency threshold over this index alone */
    uint32_t max_cnt = 0;
    {
      mm_devbuf<uint32_t> d_max; mm_devbuf<uint8_t> tmp;
      CE(d_max.reserve(1));
      const auto max_of = [&](void *t, size_t &bytes) { return cub::DeviceReduce::Max(t, bytes, cnt, d_max.get(), (int64_t)n_keys, st); };
      CE(cub_run(tmp, max_of));
      CE(cudaMemcpyAsync(&max_cnt, d_max.get(), 4, cudaMemcpyDeviceToHost, st));
      CE(cudaStreamSynchronize(st));
    }
    const uint32_t hist_n = max_cnt + 2;
    std::vector<unsigned long long> hist(hist_n);
    {
      mm_devbuf<unsigned long long> d_hist;
      CE(d_hist.reserve(hist_n));
      CE(cudaMemsetAsync(d_hist.get(), 0, (size_t)hist_n * 8, st));
      k_histogram<<<blocks(n_keys), 256, 0, st>>>(n_keys, cnt, d_hist.get(), hist_n);
      CE(cudaMemcpyAsync(hist.data(), d_hist.get(), (size_t)hist_n * 8, cudaMemcpyDeviceToHost, st));
      CE(cudaStreamSynchronize(st));
    }
    int32_t threshold = 0x7fffffff;
    { /* computeFreqHist :431-441, the same arithmetic (int64 * float / 100 -> int64; walk from the most frequent) */
      const int64_t totalUniqueMinmers = (int64_t)n_keys;
      const int64_t minmerToIgnore = totalUniqueMinmers * rule.pct / 100;
      int64_t sum = 0;
      for (int64_t f = (int64_t)hist_n - 1; f >= 0; f--) {
        if (!hist[(size_t)f]) continue;
        sum += (int64_t)hist[(size_t)f];
        if (sum < minmerToIgnore) threshold = (int32_t)f;
        else if (sum == minmerToIgnore) { threshold = (int32_t)f; break; }
        else break;
      }
      out->hist_min_count = 0; out->hist_max_count = max_cnt;
      for (uint32_t f = 0; f < hist_n; f++) if (hist[f]) { out->hist_min_count = f; out->hist_min_keys = hist[f]; break; }
      out->hist_max_keys = hist[max_cnt];
    }
    out->freq_threshold = threshold;
    k_mark_freq<<<blocks(n_keys), 256, 0, st>>>(n_keys, cnt, (uint32_t)threshold, out->is_freq.get());
  } else {
    k_mark_listed<<<blocks(n_keys), 256, 0, st>>>(n_keys, out->keys.get(), rule.d_freq, rule.n_freq, out->is_freq.get());
  }
  CE(cudaStreamSynchronize(st));
  out->counts.reset();
  /* dropFreqSeedSet: the frequent hashes leave minmerIndex (not the lookup) */
  mm_devbuf<uint32_t> keep; mm_devbuf<uint64_t> koff;
  CE(keep.reserve(n_mi)); CE(koff.reserve(n_mi + 1));
  k_keep_not_freq<<<blocks(n_mi), 256, 0, st>>>(n_mi, perm.get(), rec_key.get(), out->is_freq.get(), keep.get());
  CE(count_flags(keep.get(), koff.get(), n_mi, st, out->n_minmers));
  perm.reset(); rec_key.reset();
  CE(out->mi.reserve(out->n_minmers));
  k_compact5<<<blocks(n_mi), 256, 0, st>>>(n_mi, keep.get(), koff.get(), m.view(), out->mi.view());
  CE(cudaGetLastError());
  CE(cudaStreamSynchronize(st));
  return MM_OK;
}

/* the listed frequent hashes (rule.n_freq > 0) that the shard's keys lack: appended after them as frequent keys with no
 * points, so that every shard drops them */
int append_absent(const mm_freq_rule &rule, cudaStream_t st, mm_built_index *out, std::string &err)
{
  const uint64_t nf = rule.n_freq, n_keys = out->n_keys;
  mm_devbuf<uint32_t> absent; mm_devbuf<uint64_t> at;
  CE(absent.reserve(nf)); CE(at.reserve(nf + 1));
  k_flag_absent<<<blocks(nf), 256, 0, st>>>(nf, rule.d_freq, out->keys.get(), n_keys, absent.get());
  uint64_t n_abs = 0;
  CE(count_flags(absent.get(), at.get(), nf, st, n_abs));
  if (!n_abs) return MM_OK;
  CE(out->keys.reserve_keep(n_keys + n_abs, n_keys, st)); CE(out->offs.reserve_keep(n_keys + n_abs + 1, n_keys, st));
  CE(out->is_freq.reserve_keep(n_keys + n_abs, n_keys, st));
  if (!out->pts) CE(out->pts.reserve(1));
  k_append_absent<<<blocks(nf), 256, 0, st>>>(nf, rule.d_freq, absent.get(), at.get(), n_keys, out->n_points, out->keys.get(), out->offs.get(),
                                              out->is_freq.get());
  CE(cudaGetLastError());
  out->n_keys = n_keys + n_abs;
  CE(cudaMemcpyAsync(out->offs.get() + out->n_keys, &out->n_points, 8, cudaMemcpyHostToDevice, st));
  CE(cudaStreamSynchronize(st));
  return MM_OK;
}

/* ---- the index image (mm_capi.cu writes it from these) ---- */
__global__ void k_fill_death_keys(const int32_t *idx_wend, const uint64_t *contig_start, int32_t n_contigs, uint64_t n,
                                  uint64_t *keys, uint32_t *vals)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = n_contigs; /* contig of entry i: last c with contig_start[c] <= i */
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (contig_start[mid] <= i) lo = mid; else hi = mid;
  }
  keys[i] = ((uint64_t)(uint32_t)lo << 32) | (uint64_t)(uint32_t)idx_wend[i];
  vals[i] = (uint32_t)i;
}
__global__ void k_gather_death(const uint64_t *idx_hash, const uint64_t *keys_sorted, const uint32_t *vals_sorted, uint64_t n,
                               uint64_t *idx2_hash, int32_t *idx2_wend)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  idx2_hash[i] = idx_hash[vals_sorted[i]];
  idx2_wend[i] = (int32_t)(uint32_t)keys_sorted[i];
}

__global__ void k_split_minmers(const mm_minmer *aos, uint64_t n, uint64_t *hash, int32_t *wpos, int32_t *wend, int8_t *strand)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const mm_minmer m = aos[i];
  hash[i] = m.hash; wpos[i] = m.wpos; wend[i] = m.wpos_end; strand[i] = (int8_t)m.strand;
}
/* A loaded minmer list -> the builder's five record columns, each record checked against the one before it for what
 * mm_index_upload refuses: reason 1 a seqId outside [0, n_contigs), 2 out of (seqId, wpos) order, 4 a negative position.
 * The first bad record wins: *first_bad = min over them of (index << 8 | reasons). Kept apart from k_split_minmers, which
 * writes the index image (it has no seqId column) from records mm_index_upload has already checked on the host: one
 * kernel for both would change the upload path's code. */
__global__ void k_split_check(const mm_minmer *__restrict__ aos, uint64_t n, int32_t n_contigs, mm_rec_view o,
                              unsigned long long *first_bad)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const mm_minmer m = aos[i];
  o.hash[i] = m.hash; o.wpos[i] = m.wpos; o.wend[i] = m.wpos_end; o.seq[i] = m.seqId; o.strand[i] = (int8_t)m.strand;
  uint32_t why = 0;
  if (m.seqId < 0 || m.seqId >= n_contigs) why |= 1u;
  if (i > 0) {
    const int32_t ps = aos[i - 1].seqId, pw = aos[i - 1].wpos;
    if (m.seqId < ps || (m.seqId == ps && m.wpos < pw)) why |= 2u;
  }
  if (m.wpos < 0 || m.wpos_end < 0) why |= 4u;
  if (why) atomicMin(first_bad, ((unsigned long long)i << 8) | why);
}
/* the five record columns -> mm_minmer records (_pad = 0), records [first, first + n) */
__global__ void k_pack_minmers(mm_rec_view in, uint64_t first, uint64_t n, mm_minmer *out)
{
  const uint64_t *__restrict__ i_hash = in.hash; const int32_t *__restrict__ i_wpos = in.wpos, *__restrict__ i_wend = in.wend;
  const int32_t *__restrict__ i_seq = in.seq; const int8_t *__restrict__ i_strand = in.strand;
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t j = first + i;
  mm_minmer m;
  m.hash = i_hash[j]; m.wpos = i_wpos[j]; m.wpos_end = i_wend[j]; m.seqId = i_seq[j]; m.strand = i_strand[j]; m._pad = 0;
  out[i] = m;
}
__global__ void k_pack_points(const mm_ipoint *aos, uint64_t n, int32_t n_contigs, uint64_t *packed, uint32_t *err)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const mm_ipoint p = aos[i];
  if (p.seqId < 0 || p.seqId >= n_contigs || p.pos < 0) atomicOr(err, 1u);
  packed[i] = mm_pack_point(p.seqId, p.pos, p.side > 0);
}
/* keys are distinct: a slot is claimed by CAS on its value word, the key is written afterwards (no reader yet) */
__global__ void k_build_table(const uint64_t *keys, const uint64_t *offs, const uint8_t *is_freq, uint64_t n_keys, mm_tab_slot *tab,
                              int tab_log2, uint32_t *err)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_keys) return;
  uint64_t cnt = offs[i + 1] - offs[i];
  if (is_freq[i] && cnt > MM_VAL_CNT_MASK) cnt = MM_VAL_CNT_MASK; /* a frequent seed's list is never gathered: only the flag is read */
  if ((cnt == 0 && !is_freq[i]) || cnt > MM_VAL_CNT_MASK || offs[i] >= (1ULL << (64 - MM_VAL_OFF_SHIFT))) { atomicOr(err, 2u); return; }
  const uint64_t val = (offs[i] << MM_VAL_OFF_SHIFT) | (cnt << 1) | (is_freq[i] ? 1ULL : 0ULL);
  const uint32_t mask = (1u << tab_log2) - 1u;
  uint32_t slot = mm_tab_slot_of(keys[i], tab_log2);
  for (uint32_t probe = 0; probe <= mask; probe++) {
    const unsigned long long old = atomicCAS((unsigned long long *)&tab[slot].val, 0ULL, (unsigned long long)val);
    if (old == 0ULL) { tab[slot].key = keys[i]; return; }
    slot = (slot + 1) & mask;
  }
  atomicOr(err, 2u);
}
/* duplicates would occupy two slots: detect them after the build */
__global__ void k_check_table_dups(const mm_tab_slot *tab, int tab_log2, uint32_t *err)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t slots = 1ULL << tab_log2;
  if (i >= slots || tab[i].val == 0) return;
  const uint32_t mask = (uint32_t)(slots - 1);
  uint32_t j = ((uint32_t)i + 1) & mask;
  while (tab[j].val != 0) { /* the probe run that follows */
    if (tab[j].key == tab[i].key) { atomicOr(err, 4u); return; }
    j = (j + 1) & mask;
    if (j == (uint32_t)i) return;
  }
}

__global__ void k_count_seq(uint64_t n, const int32_t *__restrict__ seq, unsigned long long *cnt)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&cnt[seq[i]], 1ULL);
}
__global__ void k_unpack_points(uint64_t n, const uint64_t *__restrict__ pts, const uint64_t *__restrict__ keys, const uint64_t *__restrict__ offs,
                                uint64_t n_keys, mm_ipoint *out)
{ /* packed point -> skch::IntervalPoint (the hash comes from the key whose list the point is in) */
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t lo = 0, hi = n_keys; /* last key with offs <= i */
  while (lo + 1 < hi) { const uint64_t mid = (lo + hi) >> 1; if (offs[mid] <= i) lo = mid; else hi = mid; }
  mm_ipoint p;
  memset(&p, 0, sizeof p);
  p.pos = mm_point_pos(pts[i]); p.hash = keys[lo]; p.seqId = mm_point_seq(pts[i]); p.side = mm_point_open(pts[i]) ? 1 : -1;
  out[i] = p;
}

} // namespace

int mm_build_index_device(const mm_params &p, const uint8_t *d_seq, const uint64_t *h_contig_off, int32_t n_contigs,
                          const mm_freq_rule &rule, bool keep_unfiltered, cudaStream_t st, int sm_count, mm_built_index *out,
                          std::string &err)
{
  *out = mm_built_index{};
  if (!mm_sketch_kmer_supported(p.kmer_size)) { err = "k-mer size not compiled in"; return MM_EINVAL; }
  stage_events ev;
  CE(ev.create());
  cudaEventRecord(ev.e[0], st);
  int rc;
  chunk_plan plan;
  if ((rc = plan_chunks(p.kmer_size, h_contig_off, n_contigs, plan, err)) != MM_OK) return rc;
  out->n_chunks = (uint32_t)plan.chunks.size();
  {
    raw_records raw;
    if ((rc = scan_windows(p, d_seq, h_contig_off, n_contigs, plan, st, sm_count, raw, out, err)) != MM_OK) return rc;
    cudaEventRecord(ev.e[1], st);
    mm_rec_cols m; /* minmerIndex before the frequent-seed drop */
    uint64_t n_mi = 0;
    if ((rc = expand_and_sort(raw, n_contigs, p.seg_length, st, m, n_mi, err)) != MM_OK) return rc;
    out->n_minmers_before_filter = n_mi;
    cudaEventRecord(ev.e[2], st);
    if (n_mi) {
      mm_devbuf<uint32_t> perm; mm_devbuf<uint64_t> rec_key;
      if ((rc = index_lookup(m, n_mi, st, perm, rec_key, out, err)) != MM_OK) return rc;
      if (rule.mode == mm_freq_rule::COUNT_ONLY) {
        CE(cudaStreamSynchronize(st));
        out->offs.reset(); out->pts.reset(); out->is_freq.reset();
        return MM_OK;
      }
      if ((rc = frequency_filter(rule, m, n_mi, perm, rec_key, st, out, err)) != MM_OK) return rc;
    }
    if (keep_unfiltered) out->mi_unfiltered = std::move(m);
  }
  if (rule.mode == mm_freq_rule::LISTED && rule.n_freq && (rc = append_absent(rule, st, out, err)) != MM_OK) return rc;
  cudaEventRecord(ev.e[3], st);
  CE(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&out->ms_scan, ev.e[0], ev.e[1]);
  cudaEventElapsedTime(&out->ms_post, ev.e[1], ev.e[2]);
  cudaEventElapsedTime(&out->ms_lookup, ev.e[2], ev.e[3]);
  return MM_OK;
}

int mm_build_index_from_records(const mm_minmer *aos, int aos_on_device, uint64_t n, int32_t n_contigs, float kmer_pct_threshold,
                                bool keep_unfiltered, cudaStream_t st, mm_built_index *out, std::string &err)
{
  *out = mm_built_index{};
  if (n >= (1ULL << 32)) { err = "more than 2^32 minmer records"; return MM_EINVAL; }
  stage_events ev;
  CE(ev.create());
  cudaEventRecord(ev.e[0], st);
  mm_rec_cols m; /* the records, before the frequent-seed drop */
  if (n) {
    mm_devbuf<mm_minmer> staged; /* freed before the lookup, whose temporaries are larger */
    if (!aos_on_device) {
      CE(staged.reserve(n));
      CE(cudaMemcpyAsync(staged.get(), aos, n * sizeof(mm_minmer), cudaMemcpyHostToDevice, st));
    }
    const mm_minmer *d_aos = aos_on_device ? aos : staged.get();
    mm_devbuf<unsigned long long> d_bad;
    CE(d_bad.reserve(1));
    CE(cudaMemsetAsync(d_bad.get(), 0xff, 8, st));
    CE(m.reserve(n));
    k_split_check<<<blocks(n), 256, 0, st>>>(d_aos, n, n_contigs, m.view(), d_bad.get());
    CE(cudaGetLastError());
    unsigned long long bad = 0;
    CE(cudaMemcpyAsync(&bad, d_bad.get(), 8, cudaMemcpyDeviceToHost, st));
    CE(cudaStreamSynchronize(st));
    if (bad != ~0ULL) { /* refused before any kernel indexes anything by seqId */
      const unsigned long long i = bad >> 8;
      mm_minmer r;
      CE(cudaMemcpyAsync(&r, d_aos + i, sizeof r, cudaMemcpyDeviceToHost, st));
      CE(cudaStreamSynchronize(st));
      char buf[256];
      if (bad & 1u)
        snprintf(buf, sizeof buf, "record %llu: seqId %d is not a contig of this reference (%d contigs)", i, r.seqId, n_contigs);
      else if (bad & 4u)
        snprintf(buf, sizeof buf, "record %llu: negative position (wpos %d, wpos_end %d)", i, r.wpos, r.wpos_end);
      else
        snprintf(buf, sizeof buf, "record %llu (seqId %d, wpos %d) is out of (seqId, wpos) order", i, r.seqId, r.wpos);
      err = buf;
      return MM_EINVAL;
    }
  }
  out->n_minmers_before_filter = n;
  cudaEventRecord(ev.e[1], st); /* no window scan */
  cudaEventRecord(ev.e[2], st); /* and no record post-processing */
  if (n) {
    int rc;
    mm_devbuf<uint32_t> perm; mm_devbuf<uint64_t> rec_key;
    if ((rc = index_lookup(m, n, st, perm, rec_key, out, err)) != MM_OK) return rc;
    if ((rc = frequency_filter(mm_freq_rule::own_threshold(kmer_pct_threshold), m, n, perm, rec_key, st, out, err)) != MM_OK) return rc;
  }
  if (keep_unfiltered) out->mi_unfiltered = std::move(m);
  cudaEventRecord(ev.e[3], st);
  CE(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&out->ms_scan, ev.e[0], ev.e[1]);
  cudaEventElapsedTime(&out->ms_post, ev.e[1], ev.e[2]);
  cudaEventElapsedTime(&out->ms_lookup, ev.e[2], ev.e[3]);
  return MM_OK;
}

cudaError_t mm_pack_minmers(const mm_rec_cols &in, uint64_t first, uint64_t n, mm_minmer *out, cudaStream_t st)
{
  if (n == 0) return cudaSuccess;
  k_pack_minmers<<<blocks(n), 256, 0, st>>>(in.view(), first, n, out);
  return cudaGetLastError();
}

cudaError_t mm_upload_split_minmers(const mm_minmer *aos, uint64_t n, uint64_t *hash, int32_t *wpos, int32_t *wend, int8_t *strand,
                                    cudaStream_t st)
{
  if (n == 0) return cudaSuccess;
  k_split_minmers<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>(aos, n, hash, wpos, wend, strand);
  return cudaGetLastError();
}
cudaError_t mm_upload_pack_points(const mm_ipoint *aos, uint64_t n, int32_t n_contigs, uint64_t *packed, uint32_t *err, cudaStream_t st)
{
  if (n == 0) return cudaSuccess;
  k_pack_points<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>(aos, n, n_contigs, packed, err);
  return cudaGetLastError();
}
cudaError_t mm_upload_build_table(const uint64_t *keys, const uint64_t *offs, const uint8_t *is_freq, uint64_t n_keys, mm_tab_slot *tab,
                                  int tab_log2, uint32_t *err, cudaStream_t st)
{
  if (n_keys == 0) return cudaSuccess;
  k_build_table<<<(uint32_t)((n_keys + 255) / 256), 256, 0, st>>>(keys, offs, is_freq, n_keys, tab, tab_log2, err);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const uint64_t slots = 1ULL << tab_log2;
  k_check_table_dups<<<(uint32_t)((slots + 255) / 256), 256, 0, st>>>(tab, tab_log2, err);
  return cudaGetLastError();
}

/* per contig, entries sorted by wpos_end (stable): one device radix sort on (seqId, wpos_end) */
cudaError_t mm_build_death_order(const uint64_t *idx_hash, const int32_t *idx_wend, const uint64_t *contig_start,
                                 int32_t n_contigs, uint64_t n, uint64_t *idx2_hash, int32_t *idx2_wend, cudaStream_t st)
{
  if (n == 0) return cudaSuccess;
  if (n >= (1ULL << 32)) return cudaErrorInvalidValue;
  mm_devbuf<uint64_t> keys, keys2;
  mm_devbuf<uint32_t> vals, vals2;
  mm_devbuf<uint8_t> tmp;
  cudaError_t e;
  if ((e = keys.reserve(n)) != cudaSuccess || (e = keys2.reserve(n)) != cudaSuccess || (e = vals.reserve(n)) != cudaSuccess ||
      (e = vals2.reserve(n)) != cudaSuccess)
    return e;
  const uint32_t grid = (uint32_t)((n + 255) / 256);
  k_fill_death_keys<<<grid, 256, 0, st>>>(idx_wend, contig_start, n_contigs, n, keys.get(), vals.get());
  int end_bit = 32;
  while ((1LL << (end_bit - 32)) < (long long)n_contigs + 1) end_bit++;
  e = cub_run(tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceRadixSort::SortPairs(t, bytes, keys.get(), keys2.get(), vals.get(), vals2.get(), (int64_t)n, 0, end_bit, st);
  });
  if (e == cudaSuccess) k_gather_death<<<grid, 256, 0, st>>>(idx_hash, keys2.get(), vals2.get(), n, idx2_hash, idx2_wend);
  const cudaError_t s = cudaStreamSynchronize(st); /* before the temporaries go */
  return e != cudaSuccess ? e : s != cudaSuccess ? s : cudaGetLastError();
}
cudaError_t mm_index_count_seq(uint64_t n, const int32_t *seq, unsigned long long *cnt, cudaStream_t st)
{
  k_count_seq<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>(n, seq, cnt);
  return cudaGetLastError();
}
cudaError_t mm_index_unpack_points(uint64_t n, const uint64_t *pts, const uint64_t *keys, const uint64_t *offs, uint64_t n_keys,
                                   mm_ipoint *out, cudaStream_t st)
{
  k_unpack_points<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>(n, pts, keys, offs, n_keys, out);
  return cudaGetLastError();
}
