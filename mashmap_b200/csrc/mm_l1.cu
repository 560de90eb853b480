/*
 * mm_l1.cu -- K2: L1 candidate regions of every query segment.
 *
 * Replaces, per segment (rows a4-a10 of SURVEY 8(a)):
 *   the frequent-seed removal of Map::getSeedHits                  computeMap.hpp:834-839
 *   Map::getSeedIntervalPoints (hash-map probes + k-way heap merge) computeMap.hpp:856-912
 *   Stat::estimateMinimumHitsRelaxed (host table, indexed by Q.sketchSize)   :1144
 *   Map::computeL1CandidateRegions (two sweeps + cluster join)       computeMap.hpp:915-1116
 *   the per-reference-group loop of Map::doL1Mapping                 computeMap.hpp:1146-1165
 *
 * The reference merges the per-hash point lists with a heap; only the final order
 * (IntervalPoint::operator<, base_types.hpp:75-78) matters, so the points are gathered in any order
 * and sorted (bitonic). The two sweeps are restated in the stateless form of SURVEY A.5:
 *   groups   = maximal runs of consecutive points with equal pos (seqId is NOT compared, :1047,:1051)
 *   O_g      = #OPEN in points up to the end of group g
 *              - #CLOSE among points whose (seqId,pos) <= (seqId,pos) of the group's FIRST point
 *              (the trailing iterator of :1033-1046 with windowLen == 0)
 *   best     = max_g O_g (sweep #1, :948-983); return early if best < minimumHits (:987-990);
 *              HG filter raises minimumHits to sketchCutoffs[int(min(best,Q.s)/max(1,s/1000))] (:992-997)
 *   sweep #2 tests, at each group, the overlap after the PREVIOUS group (:1026-1027,:1062), so every
 *   group but the last is a candidate position iff O_g >= minimumHits; maximal stretches of flagged
 *   consecutive groups on one contig become {seqId, first pos, last pos, max O} (:1065-1098,
 *   stage2_full_scan is always true), and stretches closer than segLength are joined (:1102-1115).
 *
 * One code, two launch shapes (template parameter NT = threads that cooperate on one segment):
 *   k_l1_warp  NT = 32: ONE WARP per segment, no block barriers (warp shuffles / __syncwarp only), points sorted in
 *              that warp's shared memory (<= 512 points). Segments with more points are pushed on a list ...
 *   k_l1_cta   NT = 128: ... and done by one CTA each: 2048 points in shared memory, more in a per-CTA global
 *              scratch slice or a bump-allocated pool (the host grows the pool and re-runs if it is exhausted).
 * windowLen (computeMap.hpp:933) is 0 for every fragment of a split read and for reads no longer than segLength.
 * A fragment longer than segLength (an unsplit query, --noSplit) has windowLen = len - segLength > 0: the two kernels above
 * leave it alone and k_l1_long (one CTA per such fragment) runs the same steps 1-3 -- with every point's hit (= its
 * query hash) sorted along -- and then the two sweeps of computeMap.hpp:946-1116 literally, with hash_to_freq as one
 * counter per hit (every point's hash is a query-sketch hash). These fragments are few and have about as many points
 * as a segment, so one thread runs the sweeps.
 */
#include <algorithm>

#include "mm_internal.h"

namespace {

constexpr int L1_LOCAL_CANDS_CTA = 64;
constexpr int L1_LOCAL_CANDS_WARP = 8;
constexpr int L1_CTA_POINTS = 2048;  /* NT = 128: points handled in shared memory; more -> global scratch */
constexpr int L1_WARP_POINTS = 512;  /* NT = 32 */
constexpr int L1_WARPS_PER_CTA = 2;  /* k_l1_warp: warps (= segments in flight) per CTA */

struct l1_hit {
  uint64_t off;
  uint32_t cnt;
  uint32_t dst; /* exclusive prefix of cnt */
};

template <int NT>
struct grp {
  static __device__ __forceinline__ int tid() { return NT == 32 ? (int)(threadIdx.x & 31) : (int)threadIdx.x; }
  static __device__ __forceinline__ void sync()
  {
    if (NT == 32) __syncwarp(); else __syncthreads();
  }
};

/* exclusive prefix over the group; total = group sum */
template <int NT>
__device__ __forceinline__ uint32_t group_exclusive_scan(uint32_t v, uint32_t *warp_sums, uint32_t &total)
{
  const int lane = threadIdx.x & 31;
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (NT == 32) {
    total = __shfl_sync(0xffffffffu, incl, 31);
    return incl - v;
  }
  const int wid = threadIdx.x >> 5;
  if (lane == 31) warp_sums[wid] = incl;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < (NT + 31) / 32; w++) {
    const uint32_t s = warp_sums[w];
    if (w < wid) base += s;
    tot += s;
  }
  __syncthreads();
  total = tot;
  return base + incl - v;
}

/* in-place bitonic sort of n (power of two) u64 keys by the group (shared or global memory); PAIRS: v[] moves along */
template <int NT, bool PAIRS = false>
__device__ void group_bitonic_sort(uint64_t *a, uint32_t n, uint32_t *v = nullptr)
{
  /* (a register-resident variant -- keys in lanes, exchanges by warp shuffle -- was measured slower than this one:
   * 64-bit shuffles cost two SHFL each and the selects outweigh the saved shared-memory traffic) */
  for (uint32_t k = 2; k <= n; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t t = grp<NT>::tid(); t < (n >> 1); t += NT) {
        const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1)); /* lower index of the pair */
        const uint32_t p = i | j;
        const bool up = (i & k) == 0;
        const uint64_t x = a[i], y = a[p];
        if ((x > y) == up) {
          a[i] = y; a[p] = x;
          if (PAIRS) { const uint32_t t2 = v[i]; v[i] = v[p]; v[p] = t2; }
        }
      }
      grp<NT>::sync();
    }
  }
}

struct l1_out_list {
  mm_l1_candidate *dst; /* where candidates go (shared-memory buffer or global array) */
  uint32_t cap;         /* writes beyond cap are counted but not stored */
  uint32_t n;           /* candidates produced so far */
  uint32_t segment;
};

/* sweep #2 run state (computeMap.hpp:1009-1098) and the join (:1102-1115); uniform across the walking warp */
struct l1_walk_state {
  bool in_run;
  int run_seq, run_start, run_end, run_isz;
  int prev_group;
  bool have_out;
  int out_seq, out_start, out_end, out_isz;
};

__device__ __forceinline__ void l1_emit(l1_out_list &o, int seq, int start, int end, int isz)
{
  if (o.n < o.cap && (threadIdx.x & 31) == 0) {
    mm_l1_candidate c;
    c.seqId = seq; c.rangeStartPos = start; c.rangeEndPos = end; c.intersectionSize = isz;
    c.segment = o.segment; c.first_locus = 0; c.n_loci = 0; c._pad = 0;
    o.dst[o.n] = c;
  }
  o.n++;
}

__device__ __forceinline__ void l1_close_run(l1_walk_state &w, int seg_length, l1_out_list &o)
{
  if (!w.in_run) return;
  w.in_run = false;
  if (w.have_out && w.run_seq == w.out_seq && w.run_start <= w.out_end + seg_length) {
    w.out_end = w.run_end; /* join (computeMap.hpp:1110-1114) */
    w.out_isz = max(w.out_isz, w.run_isz);
  } else {
    if (w.have_out) l1_emit(o, w.out_seq, w.out_start, w.out_end, w.out_isz);
    w.have_out = true;
    w.out_seq = w.run_seq; w.out_start = w.run_start; w.out_end = w.run_end; w.out_isz = w.run_isz;
  }
}

/* Executed by one warp. keys[0..n): sorted points of one reference group; ginfo[i] = O_g stored at
 * the last index of each group; head[i] = index of the group's first point.
 * Sweep #2 (computeMap.hpp:1009-1098) in data-parallel form, 32 points per step: every lane that ends a group knows
 * whether its group is flagged, its contig and position and -- from the neighbouring group-ending lanes, found with
 * ballots -- whether it starts or ends a run of consecutive flagged groups on one contig. The maximum overlap of a run
 * is a segmented warp max-scan. Only the ends of runs (a handful per segment) go through the sequential join logic
 * (:1102-1115); a run that is still open at the end of a step is carried to the next one. */
__device__ void l1_walk(const uint64_t *keys, const uint32_t *ginfo, const uint32_t *head, uint32_t n, int mh,
                        int seg_length, l1_out_list &o)
{
  const int lane = threadIdx.x & 31;
  const uint32_t FULL = 0xffffffffu;
  l1_walk_state w;
  w.in_run = false; w.have_out = false; w.prev_group = -2;
  w.run_seq = w.run_start = w.run_end = w.run_isz = 0;
  w.out_seq = w.out_start = w.out_end = w.out_isz = 0;
  for (uint32_t base = 0; base < n; base += 32) {
    const uint32_t i = base + lane;
    bool last_of_group = false, flagged = false;
    int O = 0, seq = 0, pos = 0;
    if (i < n) {
      last_of_group = (i + 1 == n) || (mm_point_pos(keys[i + 1]) != mm_point_pos(keys[i]));
      if (last_of_group) {
        O = (int)ginfo[i];
        /* the last group is never tested (the test lags one group behind, :1026-1027,:1062) */
        flagged = (i + 1 != n) && (O >= mh);
        const uint64_t hk = keys[head[i]];
        seq = mm_point_seq(hk); pos = mm_point_pos(hk);
      }
    }
    const uint32_t glast = __ballot_sync(FULL, last_of_group);
    const uint32_t fl = __ballot_sync(FULL, flagged);
    if (glast == 0) continue; /* no group ends in these 32 points: nothing changes */
    if (fl == 0) {            /* only unflagged groups: an open run ends at the first of them */
      l1_close_run(w, seg_length, o);
      continue;
    }
    /* the group before / after this lane's group (group-ending lanes below / above) */
    const uint32_t below = glast & ((1u << lane) - 1u);
    const int pl = below ? 31 - __clz(below) : 0;
    const int pF_s = __shfl_sync(FULL, flagged ? 1 : 0, pl);
    const int pSeq_s = __shfl_sync(FULL, seq, pl);
    const bool prevF = below ? (pF_s != 0) : w.in_run;
    const int prevSeq = below ? pSeq_s : w.run_seq;
    const bool start = flagged && !(prevF && prevSeq == seq);
    const uint32_t above = glast & ~((2u << lane) - 1u);
    const int nl = above ? __ffs(above) - 1 : 0;
    const int nF_s = __shfl_sync(FULL, flagged ? 1 : 0, nl);
    const int nSeq_s = __shfl_sync(FULL, seq, nl);
    const bool endf = flagged && above != 0 && !(nF_s != 0 && nSeq_s == seq);
    /* segmented max of O over the run: segments begin at run starts and at unflagged groups */
    const uint32_t rmask = __ballot_sync(FULL, start || (last_of_group && !flagged));
    const uint32_t endmask = __ballot_sync(FULL, endf);
    const uint32_t upto = rmask & ((2u << lane) - 1u);
    const int hs = upto ? 31 - __clz(upto) : -1; /* first lane of this lane's segment; -1: it began in an earlier step */
    int v = flagged ? O : 0;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(FULL, v, off);
      if (lane >= off && lane - off >= hs) v = max(v, t);
    }
    const int sp_s = __shfl_sync(FULL, pos, hs < 0 ? 0 : hs);
    const int rs = hs >= 0 ? sp_s : w.run_start;                 /* where this lane's run began */
    const int vt = (hs < 0 && w.in_run) ? max(v, w.run_isz) : v; /* its maximum overlap so far */
    /* does the run carried in from the previous step go on through the first group that ends here? */
    const int f0 = __ffs(glast) - 1;
    const int f0_cont = __shfl_sync(FULL, (flagged && !start) ? 1 : 0, f0);
    if (w.in_run && !f0_cont) l1_close_run(w, seg_length, o);
    for (uint32_t em = endmask; em; em &= em - 1) { /* runs that end in this step, in order */
      const int e = __ffs(em) - 1;
      w.in_run = true;
      w.run_seq = __shfl_sync(FULL, seq, e);
      w.run_start = __shfl_sync(FULL, rs, e);
      w.run_end = __shfl_sync(FULL, pos, e);
      w.run_isz = __shfl_sync(FULL, vt, e);
      l1_close_run(w, seg_length, o);
    }
    /* carry: the last group that ends here leaves a run open iff it is flagged */
    const int ll = 31 - __clz(glast);
    const int c_seq = __shfl_sync(FULL, seq, ll), c_start = __shfl_sync(FULL, rs, ll), c_end = __shfl_sync(FULL, pos, ll),
              c_isz = __shfl_sync(FULL, vt, ll);
    if ((fl >> ll) & 1u) {
      w.in_run = true;
      w.run_seq = c_seq; w.run_start = c_start; w.run_end = c_end; w.run_isz = c_isz;
    } else {
      w.in_run = false;
    }
  }
  l1_close_run(w, seg_length, o);
  if (w.have_out) l1_emit(o, w.out_seq, w.out_start, w.out_end, w.out_isz);
}

template <int NT, int LOCAL>
struct l1_shared {
  uint32_t warp_sums[(NT + 31) / 32];
  uint32_t hmax[NT];
  int best;
  int fail;
  uint32_t range_end;
  uint32_t cand_base;
  unsigned long long scratch_base;
  uint32_t out_n;
  mm_l1_candidate local[LOCAL];
};

/* computeL1CandidateRegions over the sorted points keys[0..n) of ONE reference group.
 * Returns (uniformly) bestIntersectionSize; appends candidates through the group's first warp. */
template <int NT, int LOCAL>
__device__ int l1_process_range(const mm_params &prm, const mm_dev_index &ix, const uint64_t *keys, uint32_t *copn,
                                uint32_t *head, uint32_t *ginfo, uint32_t n, int qs, l1_shared<NT, LOCAL> &sh, l1_out_list &o,
                                int &mh_out)
{
  const int tid = grp<NT>::tid();
  const uint32_t chunk = (n + NT - 1) / NT;
  const uint32_t a = min(n, tid * chunk), e = min(n, a + chunk);
  if (tid == 0) sh.best = 0;
  /* inclusive count of OPEN points and head index of each position-group */
  uint32_t opens = 0, hmax = 0;
  for (uint32_t i = a; i < e; i++) {
    const uint64_t p = keys[i];
    opens += (uint32_t)mm_point_open(p);
    if (i == 0 || mm_point_pos(keys[i - 1]) != mm_point_pos(p)) hmax = i;
  }
  uint32_t dummy;
  const uint32_t po = group_exclusive_scan<NT>(opens, sh.warp_sums, dummy);
  uint32_t hd = 0;
  if (NT == 32) { /* exclusive max-scan of the head indices across lanes */
    uint32_t incl = hmax;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
      if (tid >= off) incl = max(incl, t);
    }
    hd = __shfl_up_sync(0xffffffffu, incl, 1);
    if (tid == 0) hd = 0;
  } else {
    sh.hmax[tid] = hmax;
    grp<NT>::sync();
    for (int t = 0; t < tid; t++) hd = max(hd, sh.hmax[t]);
  }
  uint32_t co = po;
  for (uint32_t i = a; i < e; i++) {
    const uint64_t p = keys[i];
    co += (uint32_t)mm_point_open(p);
    if (i == 0 || mm_point_pos(keys[i - 1]) != mm_point_pos(p)) hd = i;
    copn[i] = co;
    head[i] = hd;
  }
  grp<NT>::sync();
  /* O_g at the last index of every group */
  int best_local = 0;
  for (uint32_t i = a; i < e; i++) {
    const uint64_t p = keys[i];
    const bool last_of_group = (i + 1 == n) || (mm_point_pos(keys[i + 1]) != mm_point_pos(p));
    if (!last_of_group) continue;
    const uint32_t h0 = head[i];
    const uint64_t hk = keys[h0] >> 1; /* (seqId,pos) of the group's first point */
    uint32_t sub_end = i + 1;
    if ((p >> 1) != hk) { /* the group spans two contigs (equal pos): CLOSEs count up to the first sub-run only */
      sub_end = h0 + 1;
      while ((keys[sub_end] >> 1) == hk) sub_end++;
    }
    const uint32_t closes = sub_end - copn[sub_end - 1];
    const int O = (int)copn[i] - (int)closes;
    ginfo[i] = (uint32_t)O;
    best_local = max(best_local, O);
  }
  int best;
  if (NT == 32) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) best_local = max(best_local, __shfl_xor_sync(0xffffffffu, best_local, off));
    best = best_local;
    __syncwarp();
  } else {
    atomicMax(&sh.best, best_local);
    grp<NT>::sync();
    best = sh.best;
  }
  /* minimumHits (computeMap.hpp:1144, host table by Q.sketchSize) and the HG raise (:987-998) */
  int mh = ix.min_hits[min(qs, ix.n_min_hits - 1)];
  bool go = true;
  if (prm.stage1_topani_filter) {
    if (best < mh) go = false;
    else {
      const double denom = fmax(1.0, (double)prm.sketch_size / 1000.0);
      int ci = (int)((double)min(best, qs) / denom);
      ci = min(ci, ix.n_cutoffs - 1);
      mh = max(ix.cutoffs[ci], mh);
    }
  }
  mh_out = go ? mh : 0;
  if (go && tid < 32) l1_walk(keys, ginfo, head, n, mh, prm.seg_length, o);
  grp<NT>::sync();
  return best;
}

/* computeL1CandidateRegions (computeMap.hpp:915-1116) over the sorted points keys[0..n) of ONE reference group of a
 * fragment with windowLen > 0, literally, by ONE thread. hid[i] = the hit (query hash) of point i; freq[0..n_hits) is
 * hash_to_freq, cleared here and between the sweeps (:1003). Candidates go to o (join of :1102-1115 through
 * l1_close_run). Returns bestIntersectionSize of sweep #1 (uncapped); mh_out = minimumHits after the HG raise, 0 on the
 * early return (:987-990). */
__device__ int l1_window_range(const mm_params &prm, const mm_dev_index &ix, const uint64_t *keys, const uint32_t *hid,
                               uint32_t n, int qs, int window_len, int *freq, uint32_t n_hits, l1_out_list &o, int &mh_out)
{
  auto seq = [&](uint32_t i) { return mm_point_seq(keys[i]); };
  auto pos = [&](uint32_t i) { return mm_point_pos(keys[i]); };
  /* the trailing iterator (:946-976, :1033-1046): CLOSE points at or before lead.pos - windowLen on the lead's contig,
   * or on an earlier contig; a hash stops counting when its last open window closes */
  auto trail = [&](uint32_t &tr, uint32_t ld, int &overlap) {
    while (tr < n && ((seq(tr) == seq(ld) && pos(tr) <= pos(ld) - window_len) || seq(tr) < seq(ld))) {
      if (!mm_point_open(keys[tr]) && --freq[hid[tr]] == 0) overlap--;
      tr++;
    }
  };
  /* the leading iterator: every point of one position group (seqId not compared, :976, :1051); a hash starts counting
   * with its first open window */
  auto lead = [&](uint32_t &ld, int p, int &overlap) {
    while (ld < n && pos(ld) == p) {
      if (mm_point_open(keys[ld]) && freq[hid[ld]]++ == 0) overlap++;
      ld++;
    }
  };
  for (uint32_t j = 0; j < n_hits; j++) freq[j] = 0;
  int overlap = 0, best = 0;
  for (uint32_t tr = 0, ld = 0; ld < n;) { /* sweep #1 (:946-983) */
    trail(tr, ld, overlap);
    lead(ld, pos(ld), overlap);
    best = max(best, overlap);
  }
  int mh = ix.min_hits[min(qs, ix.n_min_hits - 1)];
  mh_out = 0;
  if (prm.stage1_topani_filter) {
    if (best < mh) return best; /* :987-990 */
    const double denom = fmax(1.0, (double)prm.sketch_size / 1000.0);
    const int ci = min((int)((double)min(best, qs) / denom), ix.n_cutoffs - 1);
    mh = max(ix.cutoffs[ci], mh); /* :992-997 */
  }
  mh_out = mh;
  for (uint32_t j = 0; j < n_hits; j++) freq[j] = 0; /* :1003 */
  /* sweep #2 (:1009-1098): the test lags one position group behind; a run is cut where the contig changes */
  l1_walk_state w;
  w.in_run = false; w.have_out = false; w.prev_group = -2;
  w.run_seq = w.run_start = w.run_end = w.run_isz = 0;
  w.out_seq = w.out_start = w.out_end = w.out_isz = 0;
  bool in_cand = false;
  int c_seq = 0, c_start = 0, c_end = 0, c_isz = 0; /* l1_out */
  int prev_seq = 0, prev_pos = 0, cur_seq = seq(0), cur_pos = pos(0);
  auto push_local = [&]() { /* localOpts.push_back(l1_out), joined on the fly (:1102-1115) */
    w.in_run = true;
    w.run_seq = c_seq; w.run_start = c_start; w.run_end = c_end; w.run_isz = c_isz;
    l1_close_run(w, prm.seg_length, o);
    c_seq = c_start = c_end = c_isz = 0; /* l1_out = L1_candidateLocus_t() */
  };
  overlap = 0;
  for (uint32_t tr = 0, ld = 0; ld < n;) {
    const int prev_overlap = overlap;
    trail(tr, ld, overlap);
    if (pos(ld) != cur_pos) {
      prev_seq = cur_seq; prev_pos = cur_pos;
      cur_seq = seq(ld); cur_pos = pos(ld);
    }
    lead(ld, cur_pos, overlap);
    if (prev_overlap >= mh) {
      if (c_seq != prev_seq && in_cand) {
        push_local();
        in_cand = false;
      }
      if (!in_cand) {
        c_start = c_end = prev_pos - window_len;
        c_seq = prev_seq;
        c_isz = prev_overlap;
        in_cand = true;
      } else { /* stage2_full_scan is always true (parseCmdArgs.hpp:590) */
        c_isz = max(c_isz, prev_overlap);
        c_end = prev_pos - window_len;
      }
    } else {
      if (in_cand) push_local();
      in_cand = false;
    }
  }
  if (in_cand) push_local();
  if (w.have_out) l1_emit(o, w.out_seq, w.out_start, w.out_end, w.out_isz);
  return best;
}

/* One segment, processed by a group of NT threads (the table values of its hashes are in b.sk_val, written by K1).
 * Returns false (NT == 32 only) if the segment has more points than the warp path holds: nothing was modified.
 * WIN: the segment is a fragment longer than seg_length (windowLen > 0, k_l1_long); without WIN such a fragment is
 * skipped (returns true, writes nothing). */
template <int NT, int LOCAL, int SMEM_POINTS, bool WIN = false>
__device__ bool l1_segment(const mm_params &prm, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t seg, l1_hit *hits,
                           uint64_t *skeys, uint32_t *scopn, uint32_t *shead, uint32_t *sginfo,
                           l1_shared<NT, LOCAL> &sh, uint32_t scratch_slot)
{
  const int S = prm.sketch_size;
  const int tid = grp<NT>::tid();
  const mm_segment sg = b.segs[seg];
  if (!WIN && sg.length > prm.seg_length) return true; /* k_l1_long's */
  const size_t sbase = (size_t)seg * (size_t)S;
  const int raw = b.seg_res[seg].sketch_raw_count;
  if (tid == 0) { sh.fail = 0; sh.cand_base = 0; sh.out_n = 0; }

  if (NT == 32) { /* pass A: count the points, so that an oversized segment can be handed over untouched */
    uint32_t m_probe = 0;
    for (int c0 = 0; c0 < raw; c0 += 32) {
      const int j = c0 + tid;
      uint64_t val = 0;
      if (j < raw) val = b.sk_val[sbase + j];
      m_probe += (val != 0 && !(val & 1ULL)) ? (uint32_t)((val >> 1) & MM_VAL_CNT_MASK) : 0u;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m_probe += __shfl_xor_sync(0xffffffffu, m_probe, off);
    if (m_probe > (uint32_t)SMEM_POINTS) return false;
    __syncwarp();
  }

  /* ---- 1. drop frequent seeds; compact the sketch in place; list the hit hashes ---- */
  uint32_t kept_total = 0; /* Q.sketchSize (computeMap.hpp:839) */
  uint32_t hit_total = 0;  /* kept hashes present in the lookup index (:878-883) */
  uint32_t m = 0;          /* interval points of those hashes */
  const uint64_t max_hash = raw > 0 ? b.sk_hash[sbase + raw - 1] : 0;
  for (int c0 = 0; c0 < raw; c0 += NT) {
    const int j = c0 + tid;
    uint64_t h = 0, val = 0;
    int2 ps = make_int2(0, 0);
    int8_t st = 0;
    bool keep = false;
    if (j < raw) {
      h = b.sk_hash[sbase + j];
      ps = b.sk_pos[sbase + j];
      st = b.sk_strand[sbase + j];
      val = b.sk_val[sbase + j];
      keep = !(val & 1ULL); /* !isFreqSeed (winSketch.hpp:506-509) */
    }
    const bool hit = keep && val != 0;
    const uint32_t cnt = hit ? (uint32_t)((val >> 1) & MM_VAL_CNT_MASK) : 0u;
    uint32_t tot_k, tot_h, tot_m;
    const uint32_t pk = group_exclusive_scan<NT>(keep ? 1u : 0u, sh.warp_sums, tot_k);
    const uint32_t ph = group_exclusive_scan<NT>(hit ? 1u : 0u, sh.warp_sums, tot_h);
    const uint32_t pm = group_exclusive_scan<NT>(cnt, sh.warp_sums, tot_m);
    if (keep) { /* destination index <= j: never overtakes the reads of a later chunk */
      b.sk_hash[sbase + kept_total + pk] = h;
      b.sk_pos[sbase + kept_total + pk] = ps;
      b.sk_strand[sbase + kept_total + pk] = st;
    }
    if (hit) {
      l1_hit hh;
      hh.off = val >> MM_VAL_OFF_SHIFT; hh.cnt = cnt; hh.dst = m + pm;
      hits[hit_total + ph] = hh;
    }
    kept_total += tot_k; hit_total += tot_h; m += tot_m;
  }
  grp<NT>::sync();

  /* ---- 2. gather the interval points (computeMap.hpp:887-907, order restored by the sort) ---- */
  uint32_t n_pow2 = 1;
  while (n_pow2 < m) n_pow2 <<= 1;
  uint64_t *keys = skeys;
  uint32_t *copn = scopn, *head = shead, *ginfo = sginfo;
  if (m > (uint32_t)SMEM_POINTS) { /* NT == 128 only (the warp path returned above) */
    const unsigned long long need = 3ULL * n_pow2; /* u64 units: keys + 3 u32 arrays */
    if (need <= b.scratch_slice) {
      keys = b.scratch + (size_t)scratch_slot * b.scratch_slice; /* this CTA's slice, reused per segment */
    } else {
      if (tid == 0) {
        const unsigned long long at = b.scratch_pool_off + atomicAdd((unsigned long long *)(b.counters + 4), need);
        if (at + need > b.scratch_cap) { sh.fail = 1; atomicExch(b.counters + 2, 1u); }
        sh.scratch_base = at;
      }
      grp<NT>::sync();
      if (!sh.fail) keys = b.scratch + sh.scratch_base;
    }
    if (keys != skeys) {
      copn = (uint32_t *)(keys + n_pow2);
      head = copn + n_pow2;
      ginfo = head + n_pow2;
    }
  }
  grp<NT>::sync();
  const bool fail = sh.fail != 0;
  uint32_t mp = 0; /* points that pass the skip predicates */
  if (!fail && m > 0) {
    for (uint32_t i = m + tid; i < n_pow2; i += NT) keys[i] = ~0ULL;
    uint32_t dropped_local = 0;
    const bool preds = prm.skip_self | prm.skip_prefix | prm.lower_triangular;
    auto admit = [&](uint64_t p) -> uint64_t { /* computeMap.hpp:891-893 */
      if (!preds) return p;
      const int rs = mm_point_seq(p);
      const bool ok = (!prm.skip_self || sg.name_id < 0 || sg.name_id != ix.contig_name_id[rs]) &&
                      (!prm.skip_prefix || ix.contig_group[rs] != sg.ref_group) &&
                      (!prm.lower_triangular || sg.seq_counter > rs);
      if (!ok) { dropped_local++; return ~0ULL; }
      return p;
    };
    if (keys == skeys) {
      /* point-parallel gather: owner[p] = hit that point p belongs to (head[] is free until the scans), then every
       * thread fetches 4 independent points per round -- the loads of a round are all in flight together */
      uint32_t *owner = head;
      for (uint32_t hi = tid; hi < hit_total; hi += NT) {
        const l1_hit hh = hits[hi];
        for (uint32_t q = 0; q < hh.cnt; q++) owner[hh.dst + q] = hi;
      }
      grp<NT>::sync();
      for (uint32_t p0 = tid; p0 < m; p0 += 4 * NT) {
        uint64_t v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const uint32_t p = p0 + u * NT;
          v[u] = ~0ULL;
          if (p < m) {
            const l1_hit hh = hits[owner[p]];
            v[u] = ix.pts[hh.off + (p - hh.dst)];
          }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const uint32_t p = p0 + u * NT;
          if (p < m) {
            keys[p] = admit(v[u]);
            if (WIN) copn[p] = owner[p]; /* the point's hit: its query hash */
          }
        }
      }
    } else {
      for (uint32_t hi = tid; hi < hit_total; hi += NT) {
        const l1_hit hh = hits[hi];
        for (uint32_t q = 0; q < hh.cnt; q++) {
          keys[hh.dst + q] = admit(ix.pts[hh.off + q]);
          if (WIN) copn[hh.dst + q] = hi;
        }
      }
    }
    uint32_t dropped;
    (void)group_exclusive_scan<NT>(dropped_local, sh.warp_sums, dropped);
    mp = m - dropped;
    grp<NT>::sync();
    /* ---- 3. sort by (seqId,pos,side); dropped points (all ones) go last; WIN: the hits (in copn) move along ---- */
    if (WIN) group_bitonic_sort<NT, true>(keys, n_pow2, copn);
    else group_bitonic_sort<NT>(keys, n_pow2);
  }

  /* ---- 4./5./6. per reference group: scans, best, threshold, walk ---- */
  int best_all = 0, mh_first = 0;
  l1_out_list out;
  out.dst = sh.local; out.cap = LOCAL; out.n = 0; out.segment = seg;
  for (int pass = 0; pass < 2; pass++) {
    uint32_t start = 0;
    bool first_range = true;
    while (start < mp) {
      uint32_t end = mp;
      if (prm.skip_prefix) { /* doL1Mapping groups points by reference prefix group (:1146-1165) */
        if (tid == 0) sh.range_end = mp;
        grp<NT>::sync();
        const int g0 = ix.contig_group[mm_point_seq(keys[start])];
        uint32_t found = mp;
        for (uint32_t i = start + 1 + tid; i < mp; i += NT)
          if (ix.contig_group[mm_point_seq(keys[i])] != g0) { found = i; break; }
        if (found < mp) atomicMin(&sh.range_end, found);
        grp<NT>::sync();
        end = sh.range_end;
        grp<NT>::sync();
      }
      int mh = 0, best = 0;
      if (WIN) { /* only thread 0's best / mh are read (the segment result below) */
        if (tid == 0)
          best = l1_window_range(prm, ix, keys + start, copn + start, end - start, (int)kept_total, sg.length - prm.seg_length,
                                 (int *)hits, hit_total, out, mh); /* the hit list is dead: its space holds hash_to_freq */
        grp<NT>::sync();
      } else {
        best = l1_process_range<NT, LOCAL>(prm, ix, keys + start, copn, head, ginfo, end - start, (int)kept_total, sh, out, mh);
      }
      if (pass == 0) {
        best_all = max(best_all, best);
        if (first_range) mh_first = mh;
      }
      first_range = false;
      start = end;
    }
    /* candidates were produced by the first warp: publish the count */
    if (tid == 0) sh.out_n = out.n;
    grp<NT>::sync();
    const uint32_t n_out = sh.out_n;
    if (pass == 0) {
      if (tid == 0) {
        uint32_t basec = 0;
        if (n_out > 0) {
          basec = atomicAdd(b.counters + 0, n_out);
          if ((unsigned long long)basec + n_out > b.cand_cap) atomicExch(b.counters + 3, 1u);
        }
        sh.cand_base = basec;
      }
      grp<NT>::sync();
      const uint32_t basec = sh.cand_base;
      const bool fits = (unsigned long long)basec + n_out <= b.cand_cap;
      if (n_out <= (uint32_t)LOCAL) {
        if (fits)
          for (uint32_t i = tid; i < n_out; i += NT) b.cands[basec + i] = sh.local[i];
        break;
      }
      if (!fits) break;
      /* rare: more candidates than the local buffer holds -> redo the walk writing to global memory */
      out.dst = b.cands + basec; out.cap = n_out; out.n = 0;
    }
  }
  if (tid == 0) {
    mm_segment_result r;
    r.sketch_max_hash = max_hash;
    r.sketch_raw_count = raw;
    r.sketch_size = (int32_t)kept_total;
    r.n_points = fail ? -1 : (int32_t)mp;
    r.minimum_hits = mh_first;
    r.best_intersection = best_all;
    r.first_candidate = sh.cand_base;
    r.n_candidates = sh.out_n;
    r._pad = 0;
    b.seg_res[seg] = r;
  }
  grp<NT>::sync();
  return true;
}

/* per-warp dynamic shared memory of k_l1_warp: keys | head | copn | ginfo | (hit list, if it does not fit) | state.
 * The hit list is dead once the points are gathered and copn / ginfo are first written by the scans after the sort, so
 * the list lives in their space when it fits (S <= 256); head is the gather's owner array and stays apart. */
__host__ __device__ inline size_t l1_warp_hits_extra(int S)
{
  const size_t need = (((size_t)S * sizeof(l1_hit) + 15) & ~(size_t)15);
  return need <= (size_t)L1_WARP_POINTS * 8 ? 0 : need;
}
__host__ __device__ inline size_t l1_warp_smem(int S)
{
  size_t o = (size_t)L1_WARP_POINTS * (8 + 4 + 4 + 4); /* keys, head, copn, ginfo */
  o += l1_warp_hits_extra(S);
  o += (sizeof(l1_shared<32, L1_LOCAL_CANDS_WARP>) + 15) & ~(size_t)15;
  return (o + 15) & ~(size_t)15;
}

/* fast path: one warp per segment; segments with more than L1_WARP_POINTS points go to slow_list */
__global__ void __launch_bounds__(L1_WARPS_PER_CTA * 32)
k_l1_warp(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t *slow_list)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char *base = smem_raw + l1_warp_smem(S) * wid;
  uint64_t *keys = (uint64_t *)base; base += (size_t)L1_WARP_POINTS * 8;
  uint32_t *head = (uint32_t *)base; base += (size_t)L1_WARP_POINTS * 4;
  uint32_t *copn = (uint32_t *)base; base += (size_t)L1_WARP_POINTS * 4;
  uint32_t *ginfo = (uint32_t *)base; base += (size_t)L1_WARP_POINTS * 4;
  l1_hit *hits = (l1_hit *)copn;
  if (l1_warp_hits_extra(S)) { hits = (l1_hit *)base; base += l1_warp_hits_extra(S); }
  l1_shared<32, L1_LOCAL_CANDS_WARP> &sh = *(l1_shared<32, L1_LOCAL_CANDS_WARP> *)base;

  for (uint32_t seg = blockIdx.x * L1_WARPS_PER_CTA + wid; seg < b.n_segs; seg += gridDim.x * L1_WARPS_PER_CTA) {
    __syncwarp();
    const bool done = l1_segment<32, L1_LOCAL_CANDS_WARP, L1_WARP_POINTS>(prm, ix, b, seg, hits, keys, copn, head, ginfo, sh, 0);
    if (!done && lane == 0) slow_list[atomicAdd(b.counters + 8, 1u)] = seg;
  }
}

/* general path: one CTA per listed segment (all segments when slow_list == nullptr) */
__global__ void __launch_bounds__(128)
k_l1_cta(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, const uint32_t *slow_list)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  l1_hit *hits = (l1_hit *)smem_raw;
  uint64_t *skeys = (uint64_t *)(smem_raw + (((size_t)S * sizeof(l1_hit) + 15) & ~(size_t)15));
  uint32_t *scopn = (uint32_t *)(skeys + L1_CTA_POINTS);
  uint32_t *shead = scopn + L1_CTA_POINTS;
  uint32_t *sginfo = shead + L1_CTA_POINTS;
  __shared__ l1_shared<128, L1_LOCAL_CANDS_CTA> sh;
  const uint32_t n_work = slow_list ? b.counters[8] : b.n_segs;
  for (uint32_t w = blockIdx.x; w < n_work; w += gridDim.x) {
    const uint32_t seg = slow_list ? slow_list[w] : w;
    l1_segment<128, L1_LOCAL_CANDS_CTA, L1_CTA_POINTS>(prm, ix, b, seg, hits, skeys, scopn, shead, sginfo, sh, blockIdx.x);
  }
}

/* fragments longer than seg_length (windowLen > 0): one CTA per listed fragment, the general path's layout and scratch
 * slices (it runs after k_l1_cta on the same stream) */
__global__ void __launch_bounds__(128)
k_l1_long(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, const mm_long_frag *__restrict__ longs, uint32_t n_long)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  l1_hit *hits = (l1_hit *)smem_raw;
  uint64_t *skeys = (uint64_t *)(smem_raw + (((size_t)S * sizeof(l1_hit) + 15) & ~(size_t)15));
  uint32_t *scopn = (uint32_t *)(skeys + L1_CTA_POINTS);
  uint32_t *shead = scopn + L1_CTA_POINTS;
  uint32_t *sginfo = shead + L1_CTA_POINTS;
  __shared__ l1_shared<128, L1_LOCAL_CANDS_CTA> sh;
  for (uint32_t w = blockIdx.x; w < n_long; w += gridDim.x)
    l1_segment<128, L1_LOCAL_CANDS_CTA, L1_CTA_POINTS, true>(prm, ix, b, longs[w].seg, hits, skeys, scopn, shead, sginfo, sh, blockIdx.x);
}

} // namespace

/* hit list | keys | copn | head | ginfo; the kernels' l1_shared is static shared memory on top */
size_t mm_l1_cta_smem(int sketch_size)
{
  const size_t smem = (((size_t)sketch_size * sizeof(l1_hit) + 15) & ~(size_t)15) + (size_t)L1_CTA_POINTS * (8 + 4 + 4 + 4);
  return smem + sizeof(l1_shared<128, L1_LOCAL_CANDS_CTA>) > MM_SMEM_PER_BLOCK ? 0 : smem;
}

/* CTAs of the persistent general-path grid (the scratch area holds one slice per CTA) */
uint32_t mm_l1_grid_size(const mm_params &p, int sm_count)
{
  const size_t smem = mm_l1_cta_smem(p.sketch_size);
  if (smem == 0) return 0;
  if (cudaFuncSetAttribute(k_l1_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 0;
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_l1_cta, 128, smem) != cudaSuccess) return 0;
  if (occ < 1) occ = 1;
  return (uint32_t)sm_count * (uint32_t)occ;
}

/* slow_list: device array of n_segs u32 (work list of the general path); counters[8] must be 0 */
cudaError_t mm_launch_l1(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, cudaStream_t st, int sm_count,
                         uint32_t *slow_list, int use_warp_path, int *n_launched)
{
  if (n_launched) *n_launched = 0;
  if (b.n_segs == 0) return cudaSuccess;
  uint32_t grid = mm_l1_grid_size(p, sm_count);
  if (grid == 0) return cudaErrorInvalidValue;
  const size_t wsmem = l1_warp_smem(p.sketch_size) * L1_WARPS_PER_CTA;
  if (!use_warp_path || !slow_list || wsmem > 227 * 1024) {
    k_l1_cta<<<min(grid, b.n_segs), 128, mm_l1_cta_smem(p.sketch_size), st>>>(p, ix, b, nullptr);
    if (n_launched) *n_launched = 1;
    return cudaGetLastError();
  }
  cudaError_t e = cudaFuncSetAttribute(k_l1_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_l1_warp, L1_WARPS_PER_CTA * 32, wsmem);
  if (e != cudaSuccess) return e;
  uint32_t wgrid = (uint32_t)sm_count * (uint32_t)max(occ, 1);
  wgrid = min(wgrid, (b.n_segs + L1_WARPS_PER_CTA - 1) / L1_WARPS_PER_CTA);
  k_l1_warp<<<wgrid, L1_WARPS_PER_CTA * 32, wsmem, st>>>(p, ix, b, slow_list);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  /* the general path reads its work count from counters[8] on the device: no host round trip in between */
  k_l1_cta<<<grid, 128, mm_l1_cta_smem(p.sketch_size), st>>>(p, ix, b, slow_list);
  if (n_launched) *n_launched = 2;
  return cudaGetLastError();
}

/* K2 of the fragments longer than seg_length (after mm_launch_l1, whose kernels skip them; the merge of their pieces in
 * K1 looked their hashes up) */
cudaError_t mm_launch_l1_long(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, const mm_long_frag *longs,
                              uint32_t n_long, cudaStream_t st, int sm_count)
{
  if (n_long == 0) return cudaSuccess;
  const uint32_t grid = mm_l1_grid_size(p, sm_count);
  if (grid == 0) return cudaErrorInvalidValue;
  const size_t smem = mm_l1_cta_smem(p.sketch_size);
  cudaError_t e = cudaFuncSetAttribute(k_l1_long, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_l1_long<<<min(grid, n_long), 128, smem, st>>>(p, ix, b, longs, n_long);
  return cudaGetLastError();
}
