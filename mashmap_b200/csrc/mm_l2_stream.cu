/*
 * mm_l2_stream.cu -- K3 (fast path): L2 windowed-MinHash scan as a merge of two sorted streams.
 *
 * Same contract as mm_l2.cu (Map::computeL2MappedRegions, reference computeMap.hpp:1275-1451, with the
 * SlideMapper of slidingMap.hpp:27-212); what changes is how the work is laid out on the GPU.
 *
 * The reference keeps the live reference minmers in a min-heap on wpos_end (computeMap.hpp:1296-1300) to find the
 * ones to evict before each insertion (:1344-1358). Because the index is static, that heap is replaced by a second
 * copy of each contig's entries sorted by wpos_end (the "death order", built once at upload): the entries evicted
 * while the scan moves from one position to the next are a contiguous run of that copy. A candidate's scan is then
 * a two-pointer merge of
 *   the insert stream  = index entries with rangeStart - L - 1 <= wpos <= rangeEnd, in wpos order, and
 *   the delete stream  = death-order entries with rangeStart < wpos_end <= rangeEnd, in wpos_end order,
 * with "delete while wpos_end <= wpos of the next insert" (the eviction rule, <=). Entries of the delete stream were
 * all inserted before they are met (wpos < wpos_end, interval length <= L), and the state after a batch of
 * evictions does not depend on their order (the pivot invariant is restored by every single operation).
 *
 * Three kernels:
 *   k_l2_ranges  one thread per candidate: the four binary searches that delimit its two streams, and the
 *                number of operation records it needs (host-free exclusive scan follows);
 *   k_l2_prep    one warp per candidate: lanes take consecutive stream entries (coalesced SoA reads), binary-search
 *                the hash in the query sketch held in shared memory (slidingMap.hpp:128-131) and write one 8-byte
 *                record {position, slot | match | vote} per operation; no-op deletes and set-up entries that are
 *                never inserted are compacted away with warp ballots;
 *   k_l2_scan    ONE LANE per candidate, 32 candidates per warp: the sequential rank/pivot state machine
 *                (insert_minmer / delete_minmer, slidingMap.hpp:125-211) and the region tracking
 *                (computeMap.hpp:1373-1450) run in registers; the per-query-hash counters are one packed 32-bit word
 *                per slot in shared memory, laid out [slot][lane] so the 32 candidates never bank-conflict.
 * Candidates that produce more loci than the fixed slots reserved per candidate are flagged and redone by the
 * general warp-per-candidate kernel of mm_l2.cu.
 */
#include <cub/cub.cuh>

#include "mm_internal.h"

namespace {

constexpr int L2S_WARPS = 4;
constexpr int L2S_THREADS = L2S_WARPS * 32;
constexpr int L2S_BUCKET_BITS = 9;
constexpr int L2S_BUCKETS = 1 << L2S_BUCKET_BITS; /* k_l2_prep: first-level table over the query sketch */
__host__ __device__ inline size_t l2_prep_tab_off(int S) { return (((size_t)L2S_WARPS * (size_t)(S + 2) * 9) + 15) & ~(size_t)15; }
constexpr int L2C_WARPS = 2;              /* k_l2_scan: warps per CTA (each warp = 32 candidates) */
constexpr int L2C_THREADS = L2C_WARPS * 32;
/* per-slot state word (16 bits): num_before_inc bits 0..10, active bit 11, strand_vote bits 12..15 (signed) */
constexpr uint32_t W_NBI_MASK = 0x7FFu;
constexpr uint32_t W_ACT = 1u << 11;

__device__ __forceinline__ int w_sv(uint32_t w) { return ((int)(w << 16)) >> 28; }
__device__ __forceinline__ uint32_t w_set_sv(uint32_t w, int sv) { return (w & 0x0FFFu) | (((uint32_t)sv & 0xFu) << 12); }

/* first index in [lo,hi) with a[i] >= v */
__device__ __forceinline__ uint64_t lower_bound_i32(const int32_t *a, uint64_t lo, uint64_t hi, int32_t v)
{
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void k_l2_ranges(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t n_cands)
{
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cands) return;
  const mm_l1_candidate cd = b.cands[c];
  const uint64_t cs = ix.contig_start[cd.seqId], ce = ix.contig_start[cd.seqId + 1];
  mm_l2_range r;
  /* firstOpenIt (computeMap.hpp:1290-1293) .. last entry with wpos <= rangeEnd (:1340) */
  r.it0 = lower_bound_i32(ix.idx_wpos, cs, ce, cd.rangeStartPos - prm.seg_length - 1);
  const uint64_t it1 = lower_bound_i32(ix.idx_wpos, r.it0, ce, cd.rangeEndPos + 1);
  /* evictions: wpos_end > rangeStart (anything smaller is never live) and <= rangeEnd (the last insert position) */
  r.d0 = lower_bound_i32(ix.idx2_wend, cs, ce, cd.rangeStartPos + 1);
  const uint64_t d1 = lower_bound_i32(ix.idx2_wend, r.d0, ce, cd.rangeEndPos + 1);
  /* a fragment longer than seg_length (windowLen > 0) is scanned by k_l2_long (mm_l2.cu): no records here */
  const bool windowed = b.segs[cd.segment].length > prm.seg_length;
  r.nI = windowed ? 0u : (uint32_t)(it1 - r.it0);
  r.nD = windowed ? 0u : (uint32_t)(d1 - r.d0);
  r.next_wpos = 0;
  if (r.nI > 0) r.next_wpos = (it1 < ce) ? ix.idx_wpos[it1] : ix.idx_wpos[it1 - 1]; /* std::next(windowIt,...) (:1387-1390) */
  r._pad = 0;
  b.l2_ranges[c] = r;
  b.l2_rec_off[c] = (uint64_t)r.nI + (uint64_t)r.nD; /* counts; scanned in place afterwards */
}

__global__ void __launch_bounds__(L2S_THREADS)
k_l2_prep(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t n_cands)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t *qhash = (uint64_t *)smem_raw + (size_t)wid * (S + 2);
  int8_t *qstr = (int8_t *)((uint64_t *)smem_raw + (size_t)L2S_WARPS * (S + 2)) + (size_t)wid * (S + 2);
  uint16_t *qtab = (uint16_t *)(smem_raw + l2_prep_tab_off(S)) + (size_t)wid * L2S_BUCKETS;
  const uint32_t FULL = 0xffffffffu;

  for (uint32_t c = blockIdx.x * L2S_WARPS + wid; c < n_cands; c += gridDim.x * L2S_WARPS) {
    const mm_l1_candidate cd = b.cands[c];
    mm_l2_range r = b.l2_ranges[c];
    const uint64_t off = b.l2_rec_off[c];
    if (off + r.nI + r.nD > b.l2_recs_cap) continue; /* host sized the buffer from the scan; cannot happen */
    const int n = b.seg_res[cd.segment].sketch_size;
    const size_t sbase = (size_t)cd.segment * (size_t)S;
    __syncwarp();
    for (int j = lane; j < n; j += 32) {
      qhash[j + 1] = b.sk_hash[sbase + j];
      qstr[j + 1] = b.sk_strand[sbase + j];
    }
    if (lane == 0) qhash[n + 1] = ~0ULL; /* sentinel: the forward walk below needs no bound test */
    __syncwarp();
    /* first-level table of the lower_bound over q_1..q_n (slidingMap.hpp:128-131): the sketch holds the n smallest
     * hashes of the segment, roughly uniform below q_n, so bucket = hash >> shift (shift puts q_n in the top half of the
     * table) leaves less than one sketch entry per bucket on average; qtab[b] = first j whose bucket is >= b. */
    const uint64_t qmax = n > 0 ? qhash[n] : 0ULL;
    const int shift = max(0, 64 - __clzll((long long)qmax) - L2S_BUCKET_BITS);
    for (int j = lane + 1; j <= n; j += 32) {
      const int bj = (int)(qhash[j] >> shift);
      const int bp = j == 1 ? -1 : (int)(qhash[j - 1] >> shift);
      for (int x = bp + 1; x <= bj; x++) qtab[x] = (uint16_t)j;
    }
    for (int x = (n > 0 ? (int)(qmax >> shift) + 1 : 0) + lane; x < L2S_BUCKETS; x += 32) qtab[x] = (uint16_t)(n + 1);
    __syncwarp();
    auto q_lower_bound = [&](uint64_t h) -> int {
      const uint64_t bk = h >> shift;
      if (bk >= (uint64_t)L2S_BUCKETS) return n + 1;
      int a = (int)qtab[bk];
      while (qhash[a] < h) a++;
      return a;
    };
    uint2 *out = b.l2_recs + off;
    /* Both streams are read one 32-entry chunk ahead: the loads of chunk i+1 are issued before chunk i is looked up,
     * compacted and stored (the stores keep the compiler from hoisting them by itself), so a warp always has a chunk of
     * index entries in flight -- the kernel was bound by the latency of these loads (73 % long-scoreboard stalls). The
     * wpos_end and strand of an insert entry are loaded with it, needed or not. */
    /* ---- insert stream ---- */
    struct in_entry { uint64_t h; int32_t wpos, wend; int32_t strand; };
    auto load_in = [&](uint32_t t) {
      in_entry x; x.h = 0; x.wpos = 0; x.wend = 0; x.strand = 0;
      if (t < r.nI) {
        const uint64_t e = r.it0 + t;
        x.h = ix.idx_hash[e]; x.wpos = ix.idx_wpos[e]; x.wend = ix.idx_wend[e]; x.strand = (int32_t)ix.idx_strand[e];
      }
      return x;
    };
    uint32_t n_out = 0;
    in_entry nxt = load_in((uint32_t)lane);
    for (uint32_t t0 = 0; t0 < r.nI; t0 += 32) {
      const uint32_t t = t0 + lane;
      const in_entry en = nxt;
      nxt = load_in(t + 32u);
      bool keep = false;
      uint2 rec = make_uint2(0, 0);
      if (t < r.nI) {
        const uint64_t h = en.h;
        const int wpos = en.wpos;
        const int a = q_lower_bound(h);
        const bool match = a <= n && qhash[a] == h;
        uint32_t info = (uint32_t)a;
        if (match) {
          info |= MM_L2_MATCH;
          const int vote = (int)qstr[a] * en.strand;   /* q_strand * mi.strand (slidingMap.hpp:141) */
          info |= (uint32_t)(vote & 3) << 17;           /* 2-bit two's complement: -1, 0, +1 */
        }
        if (wpos < cd.rangeStartPos) { /* set-up entry (computeMap.hpp:1323-1338) */
          keep = en.wend > cd.rangeStartPos && a <= n;
        } else {
          keep = true; /* every main entry is an evaluation point, even when it changes nothing */
        }
        rec = make_uint2((uint32_t)wpos, info);
      }
      const uint32_t km = __ballot_sync(FULL, keep);
      if (keep) out[n_out + __popc(km & ((1u << lane) - 1u))] = rec;
      n_out += __popc(km);
    }
    const uint32_t nI2 = n_out;
    /* ---- delete stream ---- */
    struct del_entry { uint64_t h; int32_t wend; };
    auto load_del = [&](uint32_t t) {
      del_entry x; x.h = 0; x.wend = 0;
      if (t < r.nD) { const uint64_t e = r.d0 + t; x.h = ix.idx2_hash[e]; x.wend = ix.idx2_wend[e]; }
      return x;
    };
    uint2 *dout = out + nI2;
    uint32_t n_del = 0;
    del_entry dnx = load_del((uint32_t)lane);
    for (uint32_t t0 = 0; t0 < r.nD; t0 += 32) {
      const uint32_t t = t0 + lane;
      const del_entry en = dnx;
      dnx = load_del(t + 32u);
      bool keep = false;
      uint2 rec = make_uint2(0, 0);
      if (t < r.nD) {
        const int a = q_lower_bound(en.h);
        keep = a <= n; /* hashes above every query hash never touch the state (slidingMap.hpp:133-136,179-182) */
        const bool match = keep && qhash[a] == en.h;
        rec = make_uint2((uint32_t)en.wend, (uint32_t)a | (match ? MM_L2_MATCH : 0u));
      }
      const uint32_t km = __ballot_sync(FULL, keep);
      if (keep) dout[n_del + __popc(km & ((1u << lane) - 1u))] = rec;
      n_del += __popc(km);
    }
    if (lane == 0) {
      r.nI = nI2;
      r.nD = n_del;
      b.l2_ranges[c] = r;
    }
  }
}

/* order of the scan: candidates sorted by their (post-compaction) operation count, longest first, so that the 32 lanes
 * of a warp run scans of similar length */
__global__ void k_l2_order_keys(const mm_dev_batch b, uint32_t n_cands, uint32_t *keys, uint32_t *vals)
{
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cands) return;
  const mm_l2_range r = b.l2_ranges[c];
  keys[c] = min(r.nI + r.nD, 0xFFFFu);
  vals[c] = c;
}

/* One lane's sequential reader of 8-byte op records. The scan consumes a record every few hundred cycles per lane and
 * L1 is almost entirely given to shared memory, so a plain `rec = p[i]` per step would expose the full DRAM/L2 latency on
 * every step. Each lane therefore owns a ring of RING_CHUNKS 16-byte cells (2 records each) per stream in shared memory,
 * laid out [cell][lane]: cells are filled by cp.async straight from global memory (no register staging), a cell is
 * re-issued for the chunk RING_CHUNKS ahead as soon as its second record has been fetched, and the line after that is
 * prefetched into L2. Fetching a record is one LDS.64 at a computed address (an earlier version kept the chunks in
 * registers and picked the record with select chains: ~40 % of the kernel's instructions).
 * Completion: when a lane first reads chunk c+1, the cp.async groups it committed after chunk c+1's own group number at
 * least RING_CHUNKS-1 (the re-issues of this stream's next cells; groups of the other stream only add to that), so
 * `cp.async.wait_group RING_CHUNKS-1` is enough. Reads run up to 2*RING_CHUNKS+2 records past a stream's end (slack). */
constexpr int RING_CHUNKS = 4;
constexpr uint32_t RING_CELL_STRIDE = 32 * 16;                       /* one cell of every lane */
constexpr uint32_t RING_STREAM_BYTES = RING_CHUNKS * RING_CELL_STRIDE; /* 2 KB per stream per warp */

__device__ __forceinline__ void ring_issue(uint32_t sm, const uint4 *g, uint32_t chunk)
{
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n\tcp.async.commit_group;" ::"r"(sm + (chunk % RING_CHUNKS) * RING_CELL_STRIDE),
               "l"(g + chunk)
               : "memory");
}
/* sm: shared address of this lane's cell 0 of the stream; g: global address of chunk 0; ptr: next record, counted from chunk 0 */
__device__ __forceinline__ uint2 ring_fetch(uint32_t sm, const uint4 *g, uint32_t &ptr)
{
  const uint32_t chunk = ptr >> 1, within = ptr & 1u;
  if (within == 0) asm volatile("cp.async.wait_group %0;" ::"n"(RING_CHUNKS - 1) : "memory");
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(sm + (chunk % RING_CHUNKS) * RING_CELL_STRIDE + within * 8u) : "memory");
  ptr++;
  if (within) {
    ring_issue(sm, g, chunk + RING_CHUNKS);
    asm volatile("prefetch.global.L2 [%0];" ::"l"(g + chunk + RING_CHUNKS + 8));
  }
  return v;
}

struct lane_locus {
  int start, end, mean, shared, strand;
};

__global__ void __launch_bounds__(L2C_THREADS)
k_l2_scan(const mm_params prm, const mm_dev_index ix, const mm_dev_batch b, uint32_t n_cands)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = prm.sketch_size;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint16_t *words = (uint16_t *)(smem_raw + (size_t)L2C_WARPS * 2 * RING_STREAM_BYTES) + (size_t)wid * (size_t)(S + 2) * 32; /* [slot][lane] */
  const uint32_t ring_sm = (uint32_t)__cvta_generic_to_shared(smem_raw) + (uint32_t)wid * 2u * RING_STREAM_BYTES;
  const uint32_t FULL = 0xffffffffu;
  const int LPC = (int)b.l2_loci_per_cand;
  const int segL = prm.seg_length;

  for (uint32_t cbase = (blockIdx.x * L2C_WARPS + wid) * 32; cbase < n_cands; cbase += gridDim.x * L2C_WARPS * 32) {
    const bool valid = cbase + lane < n_cands;
    const uint32_t c = valid ? (b.l2_perm ? b.l2_perm[cbase + lane] : cbase + lane) : 0u;
    mm_l1_candidate cd;
    mm_l2_range r;
    r.nI = 0; r.nD = 0; r.it0 = 0; r.d0 = 0; r.next_wpos = 0;
    cd.seqId = 0; cd.rangeStartPos = 0; cd.rangeEndPos = 0; cd.segment = 0;
    int n = 0;
    if (valid) {
      cd = b.cands[c];
      r = b.l2_ranges[c];
      n = b.seg_res[cd.segment].sketch_size;
    }
    /* SlideMapper::init (slidingMap.hpp:104-121): every query slot counts itself once */
    int nmax = n;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(FULL, nmax, o));
    __syncwarp();
    for (int j = 0; j <= nmax + 1; j++) {
      uint32_t w = 1u;
      if (j == 0) w = 0u;
      if (j > n) w = W_NBI_MASK; /* beyond the sketch: rank can never fit */
      words[j * 32 + lane] = (uint16_t)w;
    }
    __syncwarp();
    int pivot = n, pivRank = n, shared = 0, votes = 0;
    int pos_votes = 0; /* votes before the deletes of the current insert's position (computeMap.hpp:1342 precedes :1344) */
    bool sv_overflow = false;
    int best = 1; /* bestSketchSize (computeMap.hpp:1317) */
    bool in_cand = false, has_back = false;
    int cur_start = 0, cur_end = 0; /* the open region */
    lane_locus back = {0, 0, 0, 0, 0};
    int n_loci = 0;
    mm_l2_locus *lout = b.loci + (size_t)c * (size_t)LPC;
    auto store = [&](int k, const lane_locus &l) {
      if (k < LPC) {
        mm_l2_locus o;
        o.seqId = cd.seqId; o.meanOptimalPos = l.mean; o.optimalStart = l.start; o.optimalEnd = l.end;
        o.sharedSketchSize = l.shared; o.strand = l.strand;
        lout[k] = o;
      }
    };
    auto push_or_merge = [&](const lane_locus &l) { /* computeMap.hpp:1417-1426, :1440-1449 */
      if (!has_back) { back = l; has_back = true; }
      else if (back.end + segL < l.start) { store(n_loci, back); n_loci++; back = l; }
      else { back.end = l.end; back.mean = (back.start + back.end) / 2; }
    };

    uint32_t i = 0, d = 0;
    /* record readers: insert stream (current + next record in registers: the next one's position is read at every
     * evaluation point) and delete stream (current record) */
    const uint32_t sm_i = ring_sm + (uint32_t)lane * 16u, sm_d = sm_i + RING_STREAM_BYTES;
    const uint64_t first_i = valid ? b.l2_rec_off[c] : 0ULL, first_d = first_i + r.nI;
    const uint4 *g_i = (const uint4 *)(b.l2_recs + (first_i & ~1ULL)), *g_d = (const uint4 *)(b.l2_recs + (first_d & ~1ULL));
    uint32_t p_i = (uint32_t)(first_i & 1ULL), p_d = (uint32_t)(first_d & 1ULL);
    asm volatile("cp.async.wait_all;" ::: "memory"); /* copies still in flight for the previous candidate's cells */
    __syncwarp();
#pragma unroll
    for (int ch = 0; ch < RING_CHUNKS; ch++) { ring_issue(sm_i, g_i, ch); ring_issue(sm_d, g_d, ch); }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    uint2 irec = ring_fetch(sm_i, g_i, p_i), inext = ring_fetch(sm_i, g_i, p_i), drec = ring_fetch(sm_d, g_d, p_d);
    while (__any_sync(FULL, i < r.nI)) {
      if (i < r.nI) {
        const int ipos = (int)irec.x;
        const bool is_main = ipos >= cd.rangeStartPos;
        const bool do_del = is_main && d < r.nD && (int)drec.x <= ipos; /* evict while wpos_end <= wpos (:1344) */
        const uint32_t info = do_del ? drec.y : irec.y;
        /* the record that replaces the consumed one, from whichever stream moves: fetched now, used at the end of the
         * step, so that its shared-memory latency runs under the update */
        uint32_t p = do_del ? p_d : p_i;
        const uint2 v = ring_fetch(do_del ? sm_d : sm_i, do_del ? g_d : g_i, p);
        const int slot = (int)(info & MM_L2_SLOT_MASK);
        const bool match = (info & MM_L2_MATCH) != 0;
        const int prev_votes = pos_votes; /* only read after an insert */
        if (slot <= n) {
          /* insert_minmer / delete_minmer (slidingMap.hpp:125-165, :171-211) as one straight-line update: the four
           * cases (insert/delete x hash in the query sketch or not) are selected with predicates, so the 32 candidates of
           * the warp do not diverge. q is the slot whose membership in the pivot prefix may change: the pivot itself on
           * an insert (it is popped when the rank overflows), the slot after it on a delete (it is pulled in when it
           * fits). words[n+1] holds an unreachable count, which stands for the reference's `pivot != end` test. */
          const uint32_t w = words[slot * 32 + lane];
          const bool le = slot <= pivot;
          const int sgn = do_del ? -1 : 1;
          const int svw = w_sv(w);
          int vote = (int)((info >> 17) & 3u);
          vote = vote == 3 ? -1 : vote;
          const int sv2 = do_del ? 0 : svw + vote;
          sv_overflow |= match && (sv2 > 7 || sv2 < -8); /* the 4-bit vote sum would wrap: the general kernel redoes the candidate */
          const uint32_t w_match = w_set_sv(do_del ? (w & ~W_ACT) : (w | W_ACT), sv2);
          const uint32_t w_plain = w + (uint32_t)sgn;
          const int pr = pivRank + (le ? sgn : 0);
          const int q = pivot + (do_del ? 1 : 0);
          uint32_t x = words[q * 32 + lane];
          if (q == slot) x = w_plain;
          const int xn = (int)(x & W_NBI_MASK), xa = (x & W_ACT) ? 1 : 0, xs = w_sv(x);
          const int mv = match ? 0 : (do_del ? ((pr + xn <= n) ? 1 : 0) : ((pr > n) ? -1 : 0));
          shared += match ? (le ? sgn : 0) : mv * xa;
          votes += match ? (le ? (do_del ? -svw : sv2) : 0) : mv * xs;
          pivRank = match ? pivRank : pr + mv * xn;
          pivot += mv;
          words[slot * 32 + lane] = (uint16_t)(match ? w_match : w_plain);
        }
        { /* region tracking at every main insert (computeMap.hpp:1373-1430), as predicated updates: the branchy form
           * (three cases, struct copies) cost a quarter of the step's instructions in moves and reconvergence points.
           * While a region is open its sharedSketchSize equals `best`, so only its start and end are kept.
           *   shared > best : l2_vec_out.clear(), a new region starts here           (:1375-1392)
           *   shared == best: the open region goes on, or a new one starts here      (:1393-1406)
           *   shared < best : an open region ends at the next position               (:1407-1427) -- the only branch */
          const bool track = !do_del && is_main;
          const int npos = (i + 1 < r.nI) ? (int)inext.x : r.next_wpos;
          const bool gt = track && shared > best, ge = track && shared >= best;
          if (track && !ge && in_cand) {
            lane_locus l;
            l.start = cur_start; l.end = npos; l.mean = (cur_start + npos) / 2; l.shared = best;
            l.strand = prev_votes >= 0 ? 1 : -1;
            push_or_merge(l);
          }
          if (gt) { n_loci = 0; has_back = false; best = shared; }
          if (ge && (gt || !in_cand)) cur_start = ipos;
          if (ge) cur_end = npos;
          if (track) in_cand = ge;
        }
        /* consume the record */
        if (do_del) { p_d = p; drec = v; d++; }
        else { p_i = p; irec = inext; inext = v; i++; pos_votes = votes; }
      }
    }
    if (valid) {
      if (in_cand) { /* computeMap.hpp:1435-1450 */
        lane_locus l;
        l.start = cur_start; l.end = cur_end; l.mean = (cur_start + cur_end) / 2; l.shared = best;
        l.strand = votes >= 0 ? 1 : -1;
        push_or_merge(l);
      }
      if (has_back) { store(n_loci, back); n_loci++; }
      if (n_loci > LPC || sv_overflow) {
        atomicAdd(&b.counters->l2_redo, 1u); /* redo by the general kernel */
        b.cands[c].first_locus = 0;
        b.cands[c].n_loci = 0xFFFFFFFFu;
      } else {
        b.cands[c].first_locus = c * (uint32_t)LPC;
        b.cands[c].n_loci = (uint32_t)n_loci;
      }
    }
  }
}

} // namespace

size_t mm_l2_scan_tmp_bytes(uint32_t n_cands)
{
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (uint64_t *)nullptr, (uint64_t *)nullptr, (int)n_cands + 1);
  return bytes;
}

cudaError_t mm_launch_l2_ranges(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands,
                                void *scan_tmp, size_t scan_tmp_bytes, cudaStream_t st)
{
  if (n_cands == 0) return cudaSuccess;
  k_l2_ranges<<<(n_cands + 127) / 128, 128, 0, st>>>(p, ix, b, n_cands);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  /* exclusive scan over n_cands+1 elements: the last one (written 0 by the caller) becomes the total */
  return cub::DeviceScan::ExclusiveSum(scan_tmp, scan_tmp_bytes, b.l2_rec_off, b.l2_rec_off, (int)n_cands + 1, st);
}

/* temp bytes needed by mm_launch_l2_order for n candidates (4 u32 arrays + the library's sort storage) */
size_t mm_l2_order_bytes(uint32_t n_cands)
{
  size_t tmp = 0;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                            (uint32_t *)nullptr, (int)n_cands, 0, 16);
  return (size_t)n_cands * 16 + 1024 + tmp;
}

/* work: mm_l2_order_bytes(n_cands) bytes; returns the permutation (device pointer inside work) in *perm */
cudaError_t mm_launch_l2_order(const mm_dev_batch &b, uint32_t n_cands, void *work, size_t work_bytes, uint32_t **perm, cudaStream_t st)
{
  uint32_t *k0 = (uint32_t *)work, *v0 = k0 + n_cands, *k1 = v0 + n_cands, *v1 = k1 + n_cands;
  void *tmp = (void *)(((uintptr_t)(v1 + n_cands) + 255) & ~(uintptr_t)255);
  size_t tmp_bytes = work_bytes - (size_t)((char *)tmp - (char *)work);
  k_l2_order_keys<<<(n_cands + 255) / 256, 256, 0, st>>>(b, n_cands, k0, v0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  *perm = v1;
  return cub::DeviceRadixSort::SortPairsDescending(tmp, tmp_bytes, k0, k1, v0, v1, (int)n_cands, 0, 16, st);
}

static size_t l2_prep_smem(const mm_params &p) { return l2_prep_tab_off(p.sketch_size) + (size_t)L2S_WARPS * L2S_BUCKETS * 2; }
static size_t l2_scan_smem(const mm_params &p) { return (size_t)L2C_WARPS * ((size_t)(p.sketch_size + 2) * 32 * 2 + 2 * RING_STREAM_BYTES); }

cudaError_t mm_launch_l2_prep(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands, cudaStream_t st,
                              int sm_count)
{
  if (n_cands == 0) return cudaSuccess;
  const size_t smem = l2_prep_smem(p);
  cudaError_t e = cudaFuncSetAttribute(k_l2_prep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_l2_prep, L2S_THREADS, smem);
  if (e != cudaSuccess) return e;
  uint32_t grid = (uint32_t)sm_count * (uint32_t)max(occ, 1);
  grid = min(grid, (n_cands + L2S_WARPS - 1) / L2S_WARPS);
  k_l2_prep<<<grid, L2S_THREADS, smem, st>>>(p, ix, b, n_cands);
  return cudaGetLastError();
}

cudaError_t mm_launch_l2_scan(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, uint32_t n_cands, cudaStream_t st,
                              int sm_count)
{
  if (n_cands == 0) return cudaSuccess;
  const size_t smem = l2_scan_smem(p);
  if (smem > 227 * 1024 || p.sketch_size > 1000) return cudaErrorInvalidValue; /* 11-bit counters: caller falls back */
  cudaError_t e = cudaFuncSetAttribute(k_l2_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_l2_scan, L2C_THREADS, smem);
  if (e != cudaSuccess) return e;
  uint32_t grid = (uint32_t)sm_count * (uint32_t)max(occ, 1);
  grid = min(grid, (n_cands + L2C_THREADS - 1) / L2C_THREADS);
  k_l2_scan<<<grid, L2C_THREADS, smem, st>>>(p, ix, b, n_cands);
  return cudaGetLastError();
}
