/*
 * mm_l2.cu -- K3: L2 windowed-MinHash scan of every L1 candidate.
 *
 * Replaces Map::computeL2MappedRegions (reference src/map/include/computeMap.hpp:1275-1451) and the
 * SlideMapper it drives (slidingMap.hpp:27-212) -- row a11 of SURVEY 8(a). For one candidate
 * {seqId, rangeStartPos, rangeEndPos} and the query sketch q_1 < ... < q_n (n = Q.sketchSize):
 *   walk minmerIndex from lower_bound((seqId, rangeStart - segLength - 1)) (:1290-1293);
 *   set-up: every entry with wpos < rangeStart and wpos_end > rangeStart becomes live (:1323-1338);
 *   main:   for every entry with wpos <= rangeEnd: evict live entries with wpos_end <= wpos
 *           (:1344-1358), insert the entry (:1365-1367), then read sharedSketchElements and track
 *           maxima / ties / merges into L2_mapLocus_t records (:1373-1450).
 * Here windowLen == 0 (a fragment no longer than segLength), so the hash_to_freq paths are dead; fragments longer than
 * segLength are scanned by k_l2_long at the end of this file.
 *
 * One warp per candidate. The SlideMapper state machine (rank/pivot bookkeeping, slidingMap.hpp:125-211)
 * is kept literally -- pivot, pivRank, sharedSketchElements, strand_votes are warp-uniform registers,
 * the per-query-hash counters live in shared memory -- and the warp parallelises what surrounds it:
 *   32 index entries are loaded per step (coalesced SoA reads) and each lane binary-searches its
 *   entry's hash in the query sketch (the std::lower_bound of slidingMap.hpp:128-131,174-177);
 *   the live set (the reference's wpos_end min-heap, computeMap.hpp:1296-1300) is an unordered slot
 *   array, one slot column per lane, scanned by all lanes at once for wpos_end <= wpos; the state after
 *   a batch of evictions does not depend on their order (the pivot invariant "largest j with
 *   rank(j) <= n" is restored by every single insert/delete).
 */
#include <cub/cub.cuh>

#include "mm_internal.h"

namespace {

constexpr int L2_WARPS = 4;
constexpr int L2_THREADS = L2_WARPS * 32;
constexpr int L2_STAGE_LOCI = 16;
constexpr int L2_LIVE_SLACK = 64;

struct l2_locus_reg {
  int start, end, mean, shared, strand;
};

/* output sink: loci 0..cap-1 are stored at dst, the rest only counted */
struct l2_sink {
  mm_l2_locus *dst;
  int cap;
  int n;          /* entries flushed to dst (excluding `back`) */
  bool has_back;
  l2_locus_reg back;
  int seqId;
};

__device__ __forceinline__ void l2_store(l2_sink &s, int k, const l2_locus_reg &r)
{
  if (k < s.cap && (threadIdx.x & 31) == 0) {
    mm_l2_locus o;
    o.seqId = s.seqId; o.meanOptimalPos = r.mean; o.optimalStart = r.start; o.optimalEnd = r.end;
    o.sharedSketchSize = r.shared; o.strand = r.strand;
    s.dst[k] = o;
  }
}
/* l2_vec_out.push_back / merge with back() (computeMap.hpp:1417-1426, :1440-1449) */
__device__ __forceinline__ void l2_push_or_merge(l2_sink &s, const l2_locus_reg &cur, int seg_length)
{
  if (!s.has_back) {
    s.back = cur; s.has_back = true;
  } else if (s.back.end + seg_length < cur.start) {
    l2_store(s, s.n, s.back);
    s.n++;
    s.back = cur;
  } else {
    s.back.end = cur.end;
    s.back.mean = (s.back.start + s.back.end) / 2;
  }
}

/* per-warp shared-memory arrays */
struct l2_warp_mem {
  uint64_t *qhash; /* [n+2]: slot 0 = dummy 0 (slidingMap.hpp:86: value-initialised element 0) */
  int *nbi;        /* num_before_inc */
  int *act;        /* active */
  int *sv;         /* strand_vote */
  int8_t *qstr;    /* q_strand */
  int *lend;       /* live set: wpos_end per slot */
  uint32_t *linfo; /* live set: slot | match<<30 */
};

struct l2_state {
  int n;        /* Q.sketchSize */
  int pivot;    /* slot index of the pivot */
  int pivRank;
  int shared;   /* sharedSketchElements */
  int votes;    /* strand_votes */
  uint64_t pivhash;
};

/* SlideMapper::insert_minmer (slidingMap.hpp:125-165); slot = lower_bound position (n+1 = end) */
__device__ __forceinline__ void l2_insert(l2_state &st, const l2_warp_mem &m, int slot, bool match, int rstrand)
{
  if (slot > st.n) return;
  const int lane = threadIdx.x & 31;
  const uint64_t hv = m.qhash[slot];
  if (match) {
    const int v2 = m.sv[slot] + (int)m.qstr[slot] * rstrand;
    __syncwarp();
    if (lane == 0) { m.act[slot] = 1; m.sv[slot] = v2; }
    if (hv <= st.pivhash) { st.shared++; st.votes += v2; }
  } else {
    const int nb_piv = m.nbi[st.pivot] + (slot == st.pivot ? 1 : 0);
    const int act_piv = m.act[st.pivot];
    const int sv_piv = m.sv[st.pivot];
    const int nb_slot = m.nbi[slot];
    __syncwarp();
    if (lane == 0) m.nbi[slot] = nb_slot + 1;
    if (hv <= st.pivhash) st.pivRank++;
    if (st.pivRank > st.n) {
      st.shared -= act_piv; st.votes -= sv_piv; st.pivRank -= nb_piv;
      st.pivot--;
      st.pivhash = m.qhash[st.pivot];
    }
  }
  __syncwarp();
}

/* SlideMapper::delete_minmer (slidingMap.hpp:171-211) */
__device__ __forceinline__ void l2_delete(l2_state &st, const l2_warp_mem &m, int slot, bool match)
{
  if (slot > st.n) return;
  const int lane = threadIdx.x & 31;
  const uint64_t hv = m.qhash[slot];
  if (match) {
    const int v = m.sv[slot];
    __syncwarp();
    if (hv <= st.pivhash) { st.shared--; st.votes -= v; }
    if (lane == 0) { m.act[slot] = 0; m.sv[slot] = 0; }
  } else {
    const int nb_slot = m.nbi[slot];
    const bool has_next = st.pivot < st.n;
    const int nxt = has_next ? st.pivot + 1 : st.pivot;
    const int nb_next = m.nbi[nxt] - (slot == nxt ? 1 : 0);
    const int act_next = m.act[nxt];
    const int sv_next = m.sv[nxt];
    __syncwarp();
    if (lane == 0) m.nbi[slot] = nb_slot - 1;
    if (hv <= st.pivhash) st.pivRank--;
    if (has_next && st.pivRank + nb_next <= st.n) {
      st.pivot = nxt;
      st.shared += act_next; st.votes += sv_next; st.pivRank += nb_next;
      st.pivhash = m.qhash[nxt];
    }
  }
  __syncwarp();
}

/* One full scan of a candidate; all lanes of the warp execute it with uniform control flow.
 * Returns the number of loci (counted even beyond sink.cap), or -1 if the live set overflowed. */
__device__ int l2_scan(const mm_params &prm, const mm_dev_index &ix, const mm_l1_candidate &cd, const l2_warp_mem &m,
                       int n, int live_cap, mm_l2_locus *dst, int cap)
{
  const int lane = threadIdx.x & 31;
  const uint32_t FULL = 0xffffffffu;
  /* SlideMapper::init (slidingMap.hpp:104-121) */
  for (int j = lane; j <= n + 1; j += 32) {
    m.nbi[j] = (j >= 1 && j <= n) ? 1 : 0;
    m.act[j] = 0;
    m.sv[j] = 0;
  }
  const int rounds = (live_cap + 31) / 32;
  __syncwarp();
  l2_state st;
  st.n = n; st.pivot = n; st.pivRank = n; st.shared = 0; st.votes = 0;
  st.pivhash = m.qhash[n];

  uint64_t used = 0; /* bit r: live slot r*32+lane holds an entry */
  int min_end = 0x7fffffff;
  bool overflow = false;

  l2_sink sink;
  sink.dst = dst; sink.cap = cap; sink.n = 0; sink.has_back = false; sink.seqId = cd.seqId;
  sink.back.start = sink.back.end = sink.back.mean = sink.back.shared = sink.back.strand = 0;

  int best = 1; /* bestSketchSize (computeMap.hpp:1317) */
  bool in_cand = false;
  l2_locus_reg cur;
  cur.start = cur.end = cur.mean = cur.shared = cur.strand = 0;

  /* firstOpenIt = lower_bound(minmerIndex, {seqId, rangeStart - segLength - 1}) (computeMap.hpp:1290-1293) */
  const uint64_t cs = ix.contig_start[cd.seqId], ce = ix.contig_start[cd.seqId + 1];
  const int first_pos = cd.rangeStartPos - prm.seg_length - 1;
  uint64_t lo = cs, hi = ce;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (ix.idx_wpos[mid] < first_pos) lo = mid + 1; else hi = mid;
  }

  bool done = false;
  for (uint64_t tb = lo; tb < ce && !done; tb += 32) {
    const uint64_t t = tb + lane;
    const bool have = t < ce;
    uint64_t eh = 0;
    int ew = 0x7fffffff, ee = 0, es = 0, enw = 0;
    if (have) {
      eh = ix.idx_hash[t];
      ew = ix.idx_wpos[t];
      ee = ix.idx_wend[t];
      es = ix.idx_strand[t];
      /* std::next(windowIt, next is on the same contig)->wpos (computeMap.hpp:1387-1390); next == end() or
       * another contig -> own wpos (SURVEY A.6) */
      enw = (t + 1 < ce) ? ix.idx_wpos[t + 1] : ew;
    }
    /* slot = lower_bound over q_1..q_n (1-based); n+1 when the hash is above every query hash */
    int slot;
    bool match = false;
    {
      int a = 1, b2 = n + 1;
      while (a < b2) {
        const int mid = (a + b2) >> 1;
        if (m.qhash[mid] < eh) a = mid + 1; else b2 = mid;
      }
      slot = a;
      match = have && slot <= n && m.qhash[slot] == eh;
    }
    const bool is_setup = have && ew < cd.rangeStartPos;
    const bool is_main = have && !is_setup && ew <= cd.rangeEndPos;
    const uint32_t setup_ins = __ballot_sync(FULL, is_setup && ee > cd.rangeStartPos);
    const uint32_t main_mask = __ballot_sync(FULL, is_main);
    const uint32_t past = __ballot_sync(FULL, have && ew > cd.rangeEndPos);
    /* entries are sorted by wpos: set-up entries precede main entries precede entries past the range */
    uint32_t work = setup_ins | main_mask;
    while (work) {
      const int l = __ffs(work) - 1;
      work &= work - 1;
      const int e_slot = __shfl_sync(FULL, slot, l);
      const bool e_match = __shfl_sync(FULL, (int)match, l) != 0;
      const int e_wpos = __shfl_sync(FULL, ew, l);
      const int e_wend = __shfl_sync(FULL, ee, l);
      const int e_str = __shfl_sync(FULL, es, l);
      const int e_nw = __shfl_sync(FULL, enw, l);
      const bool e_main = (main_mask >> l) & 1u;
      const int prev_votes = st.votes; /* computeMap.hpp:1342 */

      if (e_main && e_wpos >= min_end) {
        /* evict every live entry with wpos_end <= wpos (computeMap.hpp:1344-1358) */
        int new_min = 0x7fffffff;
        for (int r = 0; r < rounds; r++) {
          const bool live = (used >> r) & 1ULL;
          const int le = live ? m.lend[r * 32 + lane] : 0x7fffffff;
          const uint32_t li = live ? m.linfo[r * 32 + lane] : 0u;
          const bool ev = live && le <= e_wpos;
          uint32_t evm = __ballot_sync(FULL, ev);
          while (evm) {
            const int el = __ffs(evm) - 1;
            evm &= evm - 1;
            const uint32_t info = __shfl_sync(FULL, li, el);
            l2_delete(st, m, (int)(info & 0x3fffffffu), (info >> 30) & 1u);
          }
          if (ev) used &= ~(1ULL << r);
          else new_min = min(new_min, le);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) new_min = min(new_min, __shfl_xor_sync(FULL, new_min, o));
        min_end = new_min;
      }
      /* insert into the live set and the slide map (computeMap.hpp:1332-1334, :1365-1367) */
      {
        const uint64_t valid = rounds >= 64 ? ~0ULL : ((1ULL << rounds) - 1ULL);
        const uint64_t freebits = ~used & valid;
        const uint32_t can = __ballot_sync(FULL, freebits != 0);
        if (can == 0) { overflow = true; done = true; break; }
        const int wl = __ffs(can) - 1;
        if (lane == wl) {
          const int r = __ffsll((long long)freebits) - 1;
          used |= 1ULL << r;
          m.lend[r * 32 + lane] = e_wend;
          m.linfo[r * 32 + lane] = (uint32_t)e_slot | (e_match ? (1u << 30) : 0u);
        }
        min_end = min(min_end, e_wend);
        __syncwarp();
        l2_insert(st, m, e_slot, e_match, e_str);
      }
      if (!e_main) continue;

      /* region tracking (computeMap.hpp:1373-1430) */
      if (st.shared > best) {
        sink.n = 0; sink.has_back = false; /* l2_vec_out.clear() */
        in_cand = true;
        best = st.shared;
        cur.shared = st.shared;
        cur.start = e_wpos;
        cur.end = e_nw;
      } else if (st.shared == best) {
        if (!in_cand) { cur.shared = st.shared; cur.start = e_wpos; }
        in_cand = true;
        cur.end = e_nw;
      } else {
        if (in_cand) {
          cur.end = e_nw;
          cur.mean = (cur.start + cur.end) / 2;
          cur.strand = prev_votes >= 0 ? 1 : -1;
          l2_push_or_merge(sink, cur, prm.seg_length);
          cur.start = cur.end = cur.mean = cur.shared = cur.strand = 0;
        }
        in_cand = false;
      }
    }
    if (past) done = true;
  }
  if (overflow) return -1;
  if (in_cand) { /* computeMap.hpp:1435-1450 */
    cur.mean = (cur.start + cur.end) / 2;
    cur.strand = st.votes >= 0 ? 1 : -1;
    l2_push_or_merge(sink, cur, prm.seg_length);
  }
  if (sink.has_back) { l2_store(sink, sink.n, sink.back); sink.n++; }
  return sink.n;
}

__global__ void __launch_bounds__(L2_THREADS)
k_l2(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t n_cands, int live_cap, int only_flagged)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  /* per-warp region */
  const size_t per_warp = ((size_t)(S + 2) * (8 + 4 + 4 + 4 + 1) + (size_t)live_cap * 8 + L2_STAGE_LOCI * sizeof(mm_l2_locus) + 63) & ~(size_t)15;
  unsigned char *base = smem_raw + per_warp * wid;
  l2_warp_mem m;
  m.qhash = (uint64_t *)base; base += (size_t)(S + 2) * 8;
  m.nbi = (int *)base; base += (size_t)(S + 2) * 4;
  m.act = (int *)base; base += (size_t)(S + 2) * 4;
  m.sv = (int *)base; base += (size_t)(S + 2) * 4;
  m.lend = (int *)base; base += (size_t)live_cap * 4;
  m.linfo = (uint32_t *)base; base += (size_t)live_cap * 4;
  mm_l2_locus *stage = (mm_l2_locus *)base; base += L2_STAGE_LOCI * sizeof(mm_l2_locus);
  m.qstr = (int8_t *)base;

  for (uint32_t c = blockIdx.x * L2_WARPS + wid; c < n_cands; c += gridDim.x * L2_WARPS) {
    mm_l1_candidate cd = b.cands[c];
    if (only_flagged && cd.n_loci != 0xFFFFFFFFu) continue; /* overflow pass after the stream kernels (mm_l2_stream.cu) */
    const uint32_t seg = cd.segment;
    if (b.segs[seg].length > prm.seg_length) continue; /* windowLen > 0: k_l2_long's */
    const int n = b.seg_res[seg].sketch_size;
    const size_t sbase = (size_t)seg * (size_t)S;
    __syncwarp();
    for (int j = lane; j < n; j += 32) {
      m.qhash[j + 1] = b.sk_hash[sbase + j];
      m.qstr[j + 1] = b.sk_strand[sbase + j];
    }
    if (lane == 0) { m.qhash[0] = 0; m.qstr[0] = 0; m.qhash[n + 1] = ~0ULL; m.qstr[n + 1] = 0; }
    __syncwarp();
    int cnt = l2_scan(prm, ix, cd, m, n, live_cap, stage, L2_STAGE_LOCI);
    uint32_t first = 0;
    if (cnt < 0) {
      if (lane == 0) atomicExch(b.counters + 1, 2u); /* live-set overflow: reported as an error */
      cnt = 0;
    } else if (cnt > 0) {
      if (lane == 0) first = atomicAdd(b.counters + 6, (uint32_t)cnt);
      first = __shfl_sync(0xffffffffu, first, 0);
      const bool fits = (unsigned long long)first + (uint32_t)cnt <= b.loci_cap;
      if (!fits) {
        if (lane == 0) atomicMax(b.counters + 1, 1u);
      } else if (cnt <= L2_STAGE_LOCI) {
        __syncwarp();
        for (int k = lane; k < cnt; k += 32) b.loci[first + k] = stage[k];
      } else {
        /* rare: more loci than the staging area -> redo the scan writing straight to global memory */
        __syncwarp();
        (void)l2_scan(prm, ix, cd, m, n, live_cap, b.loci + first, cnt);
      }
    }
    if (lane == 0) {
      b.cands[c].first_locus = first;
      b.cands[c].n_loci = (uint32_t)cnt;
    }
  }
}

/* ---- fragments longer than seg_length (windowLen = Q.len - segLength > 0, computeMap.hpp:1306) --------------------------
 * The reference keeps, next to the heap, hash_to_freq (:1309-1367): an index entry is inserted only if its hash has no
 * entry in the heap, and the eviction loop decrements the heap FRONT's count until it is 0 before popping it, so
 * hash_to_freq[h] > 0 exactly while ONE entry of h is in the heap (its later entries only add counts that the eviction
 * drains). Restated with a table `live` keyed by hash (wpos_end of the live entry of the hash, or none):
 *   set-up (wpos < rangeStart, wpos_end > rangeStart): inserted iff the hash has no live entry -- set-up entries never
 *     evict, so only the first set-up entry of a hash counts;
 *   main (wpos <= rangeEnd + windowLen), per entry: first every live entry with wpos_end <= wpos - windowLen is deleted
 *     (:1344-1358), then the entry is inserted iff its hash has no live entry; an entry that is not inserted is not
 *     evaluated (`windowIt++; continue`, :1369-1371), but the deletions before it have happened;
 *   evaluation: optimalStart = wpos ("new best", :1386) or wpos - windowLen ("tie, not in a candidate", :1398), and
 *     optimalEnd = wpos of the next INDEX entry - windowLen (:1387-1390, :1401-1404, :1409-1412), as written there.
 * Deletions come from the death-order copy of the index (wpos_end order, mm_internal.h): the entry at the death pointer
 * with wpos_end <= wpos - windowLen deletes the live entry of its hash if that one has the same wpos_end (it is itself,
 * or an entry the reference would evict at the same moment); any live entry's own death entry lies ahead of the pointer
 * when it is inserted (its wpos_end > wpos >= every threshold passed so far). The heap pops a batch of evictions in
 * wpos_end order with ties in any order; the death order is another order of the same batch, and the state after a
 * batch of evictions does not depend on their order (see the top of this file).
 * One warp per candidate, uniform control flow: the SlideMapper state machine is l2_insert / l2_delete above, the
 * lower_bound of 32 index entries at a time is lane-parallel, and the live table -- open addressing on the hash,
 * 2 u64 per slot {hash, 1<<32 | wpos_end}, at most half full -- lives in global memory, sized per candidate by
 * k_l2_long_ranges from its number of index entries. */
constexpr uint64_t L2L_USED = 1ULL << 32;

struct l2_live_table {
  uint64_t *t;
  uint32_t mask;
  /* the slot of hash h: where it is, or the empty slot where it goes (all lanes read, the same addresses) */
  __device__ __forceinline__ uint32_t find(uint64_t h) const
  {
    uint32_t i = mm_tab_slot_of(h, 32 - __clz(mask)) & mask;
    while (true) {
      const uint64_t info = t[2 * (size_t)i + 1];
      if (!(info & L2L_USED) || t[2 * (size_t)i] == h) return i;
      i = (i + 1) & mask;
    }
  }
  __device__ __forceinline__ int wend(uint32_t i) const { return (int)(uint32_t)t[2 * (size_t)i + 1]; }
  __device__ __forceinline__ void set(uint32_t i, uint64_t h, bool is_live, int wend_) const
  {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
      t[2 * (size_t)i] = h;
      /* a hash whose entry was deleted keeps its slot (the probe sequences through it stay intact), marked not live */
      t[2 * (size_t)i + 1] = is_live ? (L2L_USED | (uint64_t)(uint32_t)wend_) : (L2L_USED | (1ULL << 33));
    }
    __syncwarp();
  }
  __device__ __forceinline__ bool is_live(uint32_t i) const
  {
    const uint64_t info = t[2 * (size_t)i + 1];
    return (info & L2L_USED) && !(info & (1ULL << 33));
  }
};

/* lower_bound over q_1..q_n (1-based); n+1 when the hash is above every query hash */
__device__ __forceinline__ int l2_slot_of(const l2_warp_mem &m, int n, uint64_t h)
{
  int a = 1, b2 = n + 1;
  while (a < b2) {
    const int mid = (a + b2) >> 1;
    if (m.qhash[mid] < h) a = mid + 1; else b2 = mid;
  }
  return a;
}

/* one windowed scan (all lanes); returns the number of loci (counted beyond cap) */
__device__ int l2_scan_long(const mm_params &prm, const mm_dev_index &ix, const mm_l1_candidate &cd, const l2_warp_mem &m, int n,
                            int window_len, l2_live_table lt, mm_l2_locus *dst, int cap)
{
  const int lane = threadIdx.x & 31;
  const uint32_t FULL = 0xffffffffu;
  for (uint32_t i = lane; i <= lt.mask; i += 32) { lt.t[2 * (size_t)i] = 0; lt.t[2 * (size_t)i + 1] = 0; }
  for (int j = lane; j <= n + 1; j += 32) { /* SlideMapper::init (slidingMap.hpp:104-121) */
    m.nbi[j] = (j >= 1 && j <= n) ? 1 : 0;
    m.act[j] = 0;
    m.sv[j] = 0;
  }
  __syncwarp();
  l2_state st;
  st.n = n; st.pivot = n; st.pivRank = n; st.shared = 0; st.votes = 0;
  st.pivhash = m.qhash[n];
  l2_sink sink;
  sink.dst = dst; sink.cap = cap; sink.n = 0; sink.has_back = false; sink.seqId = cd.seqId;
  sink.back.start = sink.back.end = sink.back.mean = sink.back.shared = sink.back.strand = 0;
  int best = 1;
  bool in_cand = false;
  l2_locus_reg cur;
  cur.start = cur.end = cur.mean = cur.shared = cur.strand = 0;

  const uint64_t cs = ix.contig_start[cd.seqId], ce = ix.contig_start[cd.seqId + 1];
  const int first_pos = cd.rangeStartPos - prm.seg_length - 1;
  const int64_t last_wpos = (int64_t)cd.rangeEndPos + window_len; /* :1340 */
  uint64_t lo = cs, hi = ce;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (ix.idx_wpos[mid] < first_pos) lo = mid + 1; else hi = mid;
  }
  uint64_t dp = cs, dh = ce; /* death pointer: first entry with wpos_end > rangeStart (nothing earlier is ever live) */
  while (dp < dh) {
    const uint64_t mid = dp + ((dh - dp) >> 1);
    if (ix.idx2_wend[mid] <= cd.rangeStartPos) dp = mid + 1; else dh = mid;
  }

  bool done = false;
  for (uint64_t tb = lo; tb < ce && !done; tb += 32) {
    const uint64_t t = tb + lane;
    const bool have = t < ce;
    uint64_t eh = 0;
    int ew = 0x7fffffff, ee = 0, es = 0, enw = 0;
    if (have) {
      eh = ix.idx_hash[t]; ew = ix.idx_wpos[t]; ee = ix.idx_wend[t]; es = ix.idx_strand[t];
      enw = (t + 1 < ce) ? ix.idx_wpos[t + 1] : ew; /* std::next(windowIt, same contig)->wpos (SURVEY A.6) */
    }
    const int slot = l2_slot_of(m, n, eh);
    const bool match = have && slot <= n && m.qhash[slot] == eh;
    const bool is_setup = have && ew < cd.rangeStartPos;
    const bool is_main = have && !is_setup && (int64_t)ew <= last_wpos;
    const uint32_t setup_mask = __ballot_sync(FULL, is_setup && ee > cd.rangeStartPos);
    const uint32_t main_mask = __ballot_sync(FULL, is_main);
    if (__ballot_sync(FULL, have && (int64_t)ew > last_wpos)) done = true;
    for (uint32_t work = setup_mask | main_mask; work; work &= work - 1) {
      const int l = __ffs(work) - 1;
      const uint64_t e_hash = __shfl_sync(FULL, eh, l);
      const int e_slot = __shfl_sync(FULL, slot, l);
      const bool e_match = __shfl_sync(FULL, (int)match, l) != 0;
      const int e_wpos = __shfl_sync(FULL, ew, l);
      const int e_wend = __shfl_sync(FULL, ee, l);
      const int e_str = __shfl_sync(FULL, es, l);
      const int e_nw = __shfl_sync(FULL, enw, l);
      const bool e_main = (main_mask >> l) & 1u;
      const int prev_votes = st.votes; /* :1342 */
      if (e_main) { /* evictions (:1344-1358) */
        const int64_t thr = (int64_t)e_wpos - window_len;
        while (dp < ce && (int64_t)ix.idx2_wend[dp] <= thr) {
          const uint64_t dhash = ix.idx2_hash[dp];
          const int dwend = ix.idx2_wend[dp];
          dp++;
          const uint32_t i = lt.find(dhash);
          if (!lt.is_live(i) || lt.wend(i) != dwend) continue;
          lt.set(i, dhash, false, 0);
          const int ds = l2_slot_of(m, n, dhash);
          l2_delete(st, m, ds, ds <= n && m.qhash[ds] == dhash);
        }
      }
      const uint32_t i = lt.find(e_hash);
      if (lt.is_live(i)) continue; /* hash_to_freq[h] > 1: not inserted, not evaluated (:1365-1371) */
      lt.set(i, e_hash, true, e_wend);
      l2_insert(st, m, e_slot, e_match, e_str);
      if (!e_main) continue;
      /* region tracking (:1373-1430) */
      if (st.shared > best) {
        sink.n = 0; sink.has_back = false; /* l2_vec_out.clear() */
        in_cand = true;
        best = st.shared;
        cur.shared = st.shared;
        cur.start = e_wpos; /* :1386, no - windowLen */
        cur.end = e_nw - window_len;
      } else if (st.shared == best) {
        if (!in_cand) { cur.shared = st.shared; cur.start = e_wpos - window_len; }
        in_cand = true;
        cur.end = e_nw - window_len;
      } else {
        if (in_cand) {
          cur.end = e_nw - window_len;
          cur.mean = (cur.start + cur.end) / 2;
          cur.strand = prev_votes >= 0 ? 1 : -1;
          l2_push_or_merge(sink, cur, prm.seg_length);
          cur.start = cur.end = cur.mean = cur.shared = cur.strand = 0;
        }
        in_cand = false;
      }
    }
  }
  if (in_cand) { /* :1435-1450 */
    cur.mean = (cur.start + cur.end) / 2;
    cur.strand = st.votes >= 0 ? 1 : -1;
    l2_push_or_merge(sink, cur, prm.seg_length);
  }
  if (sink.has_back) { l2_store(sink, sink.n, sink.back); sink.n++; }
  return sink.n;
}

/* thread per candidate: 2 * (live-table slots) u64 words for a candidate of a long fragment, 0 for the others
 * (scanned into offsets afterwards) */
__global__ void k_l2_long_ranges(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t n_cands, uint64_t *words)
{
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > n_cands) return;
  if (c == n_cands) { words[c] = 0; return; }
  const mm_l1_candidate cd = b.cands[c];
  const int len = b.segs[cd.segment].length;
  if (len <= prm.seg_length) { words[c] = 0; return; }
  const uint64_t cs = ix.contig_start[cd.seqId], ce = ix.contig_start[cd.seqId + 1];
  const int first_pos = cd.rangeStartPos - prm.seg_length - 1;
  const int64_t last_wpos = (int64_t)cd.rangeEndPos + (len - prm.seg_length);
  uint64_t lo = cs, hi = ce;
  while (lo < hi) { const uint64_t mid = lo + ((hi - lo) >> 1); if (ix.idx_wpos[mid] < first_pos) lo = mid + 1; else hi = mid; }
  uint64_t e = lo;
  hi = ce;
  while (e < hi) { const uint64_t mid = e + ((hi - e) >> 1); if ((int64_t)ix.idx_wpos[mid] <= last_wpos) e = mid + 1; else hi = mid; }
  uint64_t slots = 32;
  while (slots < 2 * (e - lo) + 2) slots <<= 1;
  words[c] = 2 * slots;
}

__global__ void __launch_bounds__(L2_THREADS)
k_l2_long(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t n_cands, const uint64_t *table_off, uint64_t *table)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t per_warp = ((size_t)(S + 2) * (8 + 4 + 4 + 4 + 1) + L2_STAGE_LOCI * sizeof(mm_l2_locus) + 63) & ~(size_t)15;
  unsigned char *base = smem_raw + per_warp * wid;
  l2_warp_mem m;
  m.qhash = (uint64_t *)base; base += (size_t)(S + 2) * 8;
  m.nbi = (int *)base; base += (size_t)(S + 2) * 4;
  m.act = (int *)base; base += (size_t)(S + 2) * 4;
  m.sv = (int *)base; base += (size_t)(S + 2) * 4;
  m.lend = nullptr; m.linfo = nullptr;
  mm_l2_locus *stage = (mm_l2_locus *)base; base += L2_STAGE_LOCI * sizeof(mm_l2_locus);
  m.qstr = (int8_t *)base;

  for (uint32_t c = blockIdx.x * L2_WARPS + wid; c < n_cands; c += gridDim.x * L2_WARPS) {
    const uint64_t t0 = table_off[c], t1 = table_off[c + 1];
    if (t1 == t0) continue; /* not a long fragment's candidate */
    const mm_l1_candidate cd = b.cands[c];
    const uint32_t seg = cd.segment;
    const int n = b.seg_res[seg].sketch_size;
    const int window_len = b.segs[seg].length - prm.seg_length;
    const size_t sbase = (size_t)seg * (size_t)S;
    __syncwarp();
    for (int j = lane; j < n; j += 32) {
      m.qhash[j + 1] = b.sk_hash[sbase + j];
      m.qstr[j + 1] = b.sk_strand[sbase + j];
    }
    if (lane == 0) { m.qhash[0] = 0; m.qstr[0] = 0; m.qhash[n + 1] = ~0ULL; m.qstr[n + 1] = 0; }
    __syncwarp();
    l2_live_table lt;
    lt.t = table + t0;
    lt.mask = (uint32_t)((t1 - t0) / 2 - 1);
    int cnt = l2_scan_long(prm, ix, cd, m, n, window_len, lt, stage, L2_STAGE_LOCI);
    uint32_t first = 0;
    if (cnt > 0) {
      if (lane == 0) first = atomicAdd(b.counters + 6, (uint32_t)cnt);
      first = __shfl_sync(0xffffffffu, first, 0);
      if ((unsigned long long)first + (uint32_t)cnt > b.loci_cap) {
        if (lane == 0) atomicMax(b.counters + 1, 1u);
      } else if (cnt <= L2_STAGE_LOCI) {
        __syncwarp();
        for (int k = lane; k < cnt; k += 32) b.loci[first + k] = stage[k];
      } else { /* more loci than the staging area: the scan again, straight to global memory */
        __syncwarp();
        (void)l2_scan_long(prm, ix, cd, m, n, window_len, lt, b.loci + first, cnt);
      }
    }
    if (lane == 0) {
      b.cands[c].first_locus = first;
      b.cands[c].n_loci = (uint32_t)cnt;
    }
  }
}

} // namespace

/* four warps of: query sketch (hash, nbi, act, sv, strand) | live set (k_l2 only) | locus staging area, as the kernels
 * lay them out. k_l2's live set is one 64-bit occupancy mask per lane (l2_scan): at most 64 x 32 entries. */
size_t mm_l2_general_smem(int sketch_size, int *live_cap)
{
  const int cap = ((sketch_size + L2_LIVE_SLACK + 31) / 32) * 32;
  if (cap > 64 * 32) return 0;
  const size_t per_warp = ((size_t)(sketch_size + 2) * (8 + 4 + 4 + 4 + 1) + (size_t)cap * 8 +
                           L2_STAGE_LOCI * sizeof(mm_l2_locus) + 63) & ~(size_t)15;
  const size_t smem = per_warp * L2_WARPS;
  if (smem > MM_SMEM_PER_BLOCK) return 0;
  if (live_cap) *live_cap = cap;
  return smem;
}

size_t mm_l2_long_smem(int sketch_size)
{
  const size_t per_warp = ((size_t)(sketch_size + 2) * (8 + 4 + 4 + 4 + 1) + L2_STAGE_LOCI * sizeof(mm_l2_locus) + 63) & ~(size_t)15;
  const size_t smem = per_warp * L2_WARPS;
  return smem > MM_SMEM_PER_BLOCK ? 0 : smem;
}

static cudaError_t launch_general(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                  cudaStream_t st, int sm_count, int only_flagged)
{
  if (n_cands == 0) return cudaSuccess;
  int live_cap = 0;
  const size_t smem = mm_l2_general_smem(p.sketch_size, &live_cap);
  if (smem == 0) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(k_l2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_l2, L2_THREADS, smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) occ = 1;
  uint32_t grid = (uint32_t)sm_count * (uint32_t)occ;
  const uint32_t need = (n_cands + L2_WARPS - 1) / L2_WARPS;
  if (grid > need) grid = need;
  k_l2<<<grid, L2_THREADS, smem, st>>>(p, ix, b, n_cands, live_cap, only_flagged);
  return cudaGetLastError();
}

/* general warp-per-candidate kernel over every candidate */
cudaError_t mm_launch_l2(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                         cudaStream_t st, int sm_count)
{
  return launch_general(p, ix, b, n_cands, st, sm_count, 0);
}

/* only the candidates the stream kernels flagged (more loci than their fixed slots) */
cudaError_t mm_launch_l2_overflow(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                  cudaStream_t st, int sm_count)
{
  return launch_general(p, ix, b, n_cands, st, sm_count, 1);
}

/* live-table offsets of the candidates of long fragments: counts, then an exclusive scan over n_cands + 1 entries
 * (table_off[n_cands] = total u64 words) */
cudaError_t mm_launch_l2_long_ranges(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                     uint64_t *table_off, void *scan_tmp, size_t scan_tmp_bytes, cudaStream_t st)
{
  k_l2_long_ranges<<<(n_cands + 1 + 127) / 128, 128, 0, st>>>(p, ix, b, n_cands, table_off);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return cub::DeviceScan::ExclusiveSum(scan_tmp, scan_tmp_bytes, table_off, table_off, (int)n_cands + 1, st);
}

/* the windowed scan of every candidate whose table_off range is not empty; loci appended at counters[6] */
cudaError_t mm_launch_l2_long(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                              const uint64_t *table_off, uint64_t *table, cudaStream_t st, int sm_count)
{
  if (n_cands == 0) return cudaSuccess;
  const size_t smem = mm_l2_long_smem(p.sketch_size);
  if (smem == 0) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(k_l2_long, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  uint32_t grid = (uint32_t)sm_count * 4u;
  const uint32_t need = (n_cands + L2_WARPS - 1) / L2_WARPS;
  if (grid > need) grid = need;
  k_l2_long<<<grid, L2_THREADS, smem, st>>>(p, ix, b, n_cands, table_off, table);
  return cudaGetLastError();
}
