/*
 * mm_align.cu -- the device path of mashmap-b200-align: edlibAlign(query, target, k, EDLIB_MODE_HW, EDLIB_TASK_PATH)
 * (reference src/common/edlib.hxx:141-260, called from computeAlignments.hpp:268) for a batch of mappings, and of
 * mashmap-b200 --align: the same call in EDLIB_MODE_NW.
 *
 * edlib bands its Myers bit-vector computation (Ukkonen); every decision it takes depends only on exact scores <= k, and
 * banded scores never underestimate, so an unbanded computation takes the same decisions (DESIGN.md section 10; pinned by
 * tests/test_align_cpu.py on the CPU restatement). Here every sweep is unbanded and exact. Rules restated:
 *   1. ed = min over target columns of the HW last-row score (-1 if > k); end = the SMALLEST column reaching it. When the
 *      query length is not a multiple of 64, edlib's padded last block also offers column -1 (empty target, score Q).
 *   2. start = end - (LARGEST position of the minimum in the SHW pass of the reversed query over the reversed target
 *      prefix [0, end]).
 *   3. path = NW of query against target[start..end] with score ed: traceback over stored blocks (move preference up,
 *      left, diagonal) when (2*8+4)*ceil(Q/64)*T + 8*T < 1 MiB, otherwise one Hirschberg split (target at T/2; first row
 *      whose forward + reverse scores sum to the score, then the -1 boundary, then the Q-1 boundary) and recursion.
 *
 * Global mode (EDLIB_MODE_NW, edlib.hxx:193-248), for jobs with mode MM_ALIGN_NW:
 *   1'. ed = the NW score at (Q-1, T-1) (-1 if k >= 0 and ed > k); start = 0, end = T-1, no SHW pass.
 *   3'. path = rule 3 over the whole target with score ed.
 *
 * Kernels, all one warp per problem with the 64-bit blocks of the query spread over the lanes (lane l owns a contiguous
 * run of blocks) and a wavefront along the target (lane l works on column s - l at step s; the horizontal carry moves
 * one lane down per step through a shuffle):
 *   k_align_hw      (a) rule 1              k_align_shw  (b) rule 2
 *   k_align_nw      (a) rule 1'
 *   k_align_hirsch  (c) one Hirschberg level: forward and reverse NW boundary columns, then the split row
 *   k_align_leaf    (d) NW with every column's blocks stored, then the traceback to edit ops
 * The host walks the levels (the next level's list keeps sub-problems in alignment order) and schedules the leaves'
 * block storage in waves under the context's scratch budget.
 *
 * Long sub-problems (max(Q, T) >= MM_ALIGN_BAND_MIN_LEN; leaves never are) run banded, one CTA per sweep, sized to the
 * band:
 *   k_band_nw       (a) rule 1' for one pass of a k schedule the host drives
 *   k_band_col      (c) one half-column of a Hirschberg node (two CTAs per node), then k_band_split for the split row
 *
 * mm_align_batch_tags formats the paths on the device instead of returning them (DESIGN.md section 10, "Tag text on
 * the device"), flat over the ops of a wave of jobs: k_tag_gather (compact the leaves), k_tag_mark + cub select (run
 * starts), k_tag_runs + cub scans (run text lengths, offsets and base positions), k_tag_jobs (job text offsets),
 * k_tag_write (one thread per output byte).
 */
#include <cstdlib>
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "../../include/mashmap_b200_align.h"
#include "mm_devbuf.h"

namespace {

constexpr unsigned FULL = 0xffffffffu;
enum { M_HW = 0, M_SHW = 1, M_COL = 2, M_STORE = 3, M_NW = 4 };

struct Prob {
  uint64_t q, t;     // forward substrings: d_q + q, d_t + t
  int32_t ql, tl;
  int32_t k;         // HW: edlib's k; Hirschberg: the sub-problem's NW score
  int32_t res;       // index of this problem's outputs
  uint64_t scratch;  // byte offset of its scratch
  uint64_t out;      // leaf: offset of its op area (ql + tl bytes)
};

__host__ __device__ inline int nblocks(int ql) { return (ql + 63) >> 6; }
__host__ __device__ inline uint64_t al16(uint64_t x) { return (x + 15) & ~(uint64_t)15; }

/* Peq[s * nb + b]: bit i set when query row 64b + i holds symbol s; rows past the query (padding) match everything.
 * The calling warp builds blocks b0, b0 + bstep, ... (the whole query by default). */
__device__ void build_peq(uint64_t *peq, const uint8_t *q, int ql, bool rev, const uint8_t *code, int nsym, int lane,
                          int b0 = 0, int bstep = 1)
{
  const int nb = nblocks(ql);
  for (int b = b0; b < nb; b += bstep) {
    const int r0 = b * 64 + lane, r1 = r0 + 32;
    const int c0 = r0 < ql ? code[rev ? q[ql - 1 - r0] : q[r0]] : -1;
    const int c1 = r1 < ql ? code[rev ? q[ql - 1 - r1] : q[r1]] : -1;
    for (int s = 0; s < nsym; s++) {
      const unsigned lo = __ballot_sync(FULL, c0 == s || c0 < 0);
      const unsigned hi = __ballot_sync(FULL, c1 == s || c1 < 0);
      if (lane == 0) peq[(size_t)s * nb + b] = ((uint64_t)hi << 32) | lo;
    }
  }
  __syncwarp();
}

/* One Myers sweep of a query (given by its Peq) over tl target columns. Block state: P / M vertical-delta words and the
 * score of the block's bottom row. M_HW / M_SHW track the last query row and return its minimum over the columns
 * (smallest column for HW, largest for SHW) in best / bestpos on every lane; M_NW tracks it the same way and returns its
 * value at the last column; M_STORE keeps every column's blocks at [c * nb + b] for the traceback. The top boundary is 0
 * for HW (free start) and +1 per column otherwise. */
template <int MODE>
__device__ void sweep(const uint64_t *peq, int ql, const uint8_t *t, int tl, bool trev, const uint8_t *code,
                      uint64_t *Ps, uint64_t *Ms, int *Ss, int lane, int &best, int &bestpos)
{
  const int nb = nblocks(ql);
  const int bpl = (nb + 31) >> 5;
  const int lanes = (nb + bpl - 1) / bpl;
  const int b0 = lane * bpl, b1 = min(nb, b0 + bpl);
  const int lastr = (ql - 1) & 63;
  const int top = MODE == M_HW ? 0 : 1;
  constexpr bool track = MODE == M_HW || MODE == M_SHW || MODE == M_NW;
  if (MODE != M_STORE)
    for (int b = b0; b < b1; b++) { Ps[b] = ~0ull; Ms[b] = 0; Ss[b] = 64 * (b + 1); }
  int row = ql;  // last query row at column -1
  best = (MODE == M_HW && (ql & 63)) ? ql : INT_MAX;
  bestpos = -1;
  int carry = 0;
  const int steps = tl + lanes - 1;
  for (int s = 0; s < steps; s++) {
    int hin = __shfl_up_sync(FULL, carry, 1);
    if (lane == 0) hin = top;
    const int c = s - lane;
    if (lane < lanes && c >= 0 && c < tl) {
      const uint64_t *pq = peq + (size_t)code[trev ? t[tl - 1 - c] : t[c]] * nb;
      int h = hin;
      for (int b = b0; b < b1; b++) {
        uint64_t Pv, Mv;
        int sc;
        if (MODE == M_STORE) {
          if (c == 0) { Pv = ~0ull; Mv = 0; sc = 64 * (b + 1); }
          else { const size_t i = (size_t)(c - 1) * nb + b; Pv = Ps[i]; Mv = Ms[i]; sc = Ss[i]; }
        } else {
          Pv = Ps[b]; Mv = Ms[b]; sc = Ss[b];
        }
        uint64_t Eq = pq[b];
        const uint64_t Xv = Eq | Mv;
        if (h < 0) Eq |= 1ull;
        const uint64_t Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
        uint64_t Ph = Mv | ~(Xh | Pv);
        uint64_t Mh = Pv & Xh;
        const int hout = (int)(Ph >> 63) - (int)(Mh >> 63);
        if (track && b == nb - 1)
          row += (int)((Ph >> lastr) & 1) - (int)((Mh >> lastr) & 1);
        Ph <<= 1;
        Mh <<= 1;
        if (h < 0) Mh |= 1ull;
        else if (h > 0) Ph |= 1ull;
        Pv = Mh | ~(Xv | Ph);
        Mv = Ph & Xv;
        sc += hout;
        if (MODE == M_STORE) {
          const size_t i = (size_t)c * nb + b;
          Ps[i] = Pv; Ms[i] = Mv; Ss[i] = sc;
        } else {
          Ps[b] = Pv; Ms[b] = Mv; Ss[b] = sc;
        }
        h = hout;
      }
      carry = h;
      if (track && b1 == nb && b0 < b1) {
        if (MODE == M_NW ? c == tl - 1 : MODE == M_HW ? row < best : row <= best) { best = row; bestpos = c; }
      }
    }
  }
  best = __shfl_sync(FULL, best, lanes - 1);
  bestpos = __shfl_sync(FULL, bestpos, lanes - 1);
  __syncwarp();
}

/* scores of every query row from a column's blocks; reversed: row r goes to out[ql - 1 - r] */
__device__ void write_column(const uint64_t *P, const uint64_t *M, const int *S, int ql, int *out, bool reversed, int lane)
{
  const int nb = nblocks(ql);
  for (int b = lane; b < nb; b += 32) {
    const uint64_t p = P[b], m = M[b];
    int v = S[b];
    for (int i = 63; i >= 0; i--) {
      const int r = b * 64 + i;
      if (r < ql) out[reversed ? ql - 1 - r : r] = v;
      v -= (int)((p >> i) & 1) - (int)((m >> i) & 1);
    }
  }
  __syncwarp();
}

struct Scratch {  // carving of one problem's scratch
  uint64_t *peq, *P, *M;
  int *S;
  __device__ Scratch(uint8_t *base, int ql, int nsym, uint64_t cols)
  {
    const int nb = nblocks(ql);
    peq = (uint64_t *)base;
    P = (uint64_t *)(base + al16((uint64_t)nsym * nb * 8));
    M = P + cols * nb;
    S = (int *)(M + cols * nb);
  }
};
__host__ __device__ inline uint64_t scratch_bytes(int ql, int nsym, uint64_t cols, uint64_t extra)
{
  const uint64_t nb = (uint64_t)nblocks(ql);
  return al16(nsym * nb * 8) + al16(cols * nb * 20) + al16(extra);
}

__global__ void k_align_hw(const Prob *probs, int n, const uint8_t *dq, const uint8_t *dt, const uint8_t *code, int nsym,
                           uint8_t *scratch, int *out_ed, int *out_end)
{
  const int w = (int)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  const Prob p = probs[w];
  Scratch sc(scratch + p.scratch, p.ql, nsym, 1);
  build_peq(sc.peq, dq + p.q, p.ql, false, code, nsym, lane);
  int best, pos;
  sweep<M_HW>(sc.peq, p.ql, dt + p.t, p.tl, false, code, sc.P, sc.M, sc.S, lane, best, pos);
  const int kk = p.k < 0 ? INT_MAX : min(p.k, p.ql);  // HW: edlib caps k at the query length (edlib.hxx:531-533)
  if (lane == 0) {
    out_ed[p.res] = best <= kk ? best : -1;
    out_end[p.res] = best <= kk ? pos : -1;
  }
}

/* rule 1': edlib's NW distance accepts the exact score when it is <= k (myersCalcEditDistanceNW, edlib.hxx:695-902) */
__global__ void k_align_nw(const Prob *probs, int n, const uint8_t *dq, const uint8_t *dt, const uint8_t *code, int nsym,
                           uint8_t *scratch, int *out_ed, int *out_end)
{
  const int w = (int)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  const Prob p = probs[w];
  Scratch sc(scratch + p.scratch, p.ql, nsym, 1);
  build_peq(sc.peq, dq + p.q, p.ql, false, code, nsym, lane);
  int best, pos;
  sweep<M_NW>(sc.peq, p.ql, dt + p.t, p.tl, false, code, sc.P, sc.M, sc.S, lane, best, pos);
  const bool ok = p.k < 0 || best <= p.k;
  if (lane == 0) {
    out_ed[p.res] = ok ? best : -1;
    out_end[p.res] = ok ? pos : -1;
  }
}

__global__ void k_align_shw(const Prob *probs, int n, const uint8_t *dq, const uint8_t *dt, const uint8_t *code, int nsym,
                            uint8_t *scratch, int *out_start)
{
  const int w = (int)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  const Prob p = probs[w];  // target = [t, t + tl) with tl = end + 1, read backwards
  Scratch sc(scratch + p.scratch, p.ql, nsym, 1);
  build_peq(sc.peq, dq + p.q, p.ql, true, code, nsym, lane);
  int best, pos;
  sweep<M_SHW>(sc.peq, p.ql, dt + p.t, p.tl, true, code, sc.P, sc.M, sc.S, lane, best, pos);
  if (lane == 0) out_start[p.res] = (p.tl - 1) - pos;
}

/* The Hirschberg split of a node from its boundary columns (left[i] = NW(query[0..i], target[0..lw)), right[i] =
 * NW(query[i..Q), target[lw..T))): the first row in ascending order whose scores sum to the node's score, then the -1
 * boundary, then the Q-1 boundary. {split row, upper-left score, lower-right score, 1}, or {0, 0, 0, 0} when no row
 * sums to the score; the same on every lane. */
__device__ int4 split_row(const int *left, const int *right, int Q, int lw, int rw, int best, int lane)
{
  int split = INT_MIN, ls = 0, rs = 0;
  for (int base = 0; base < Q - 1 && split == INT_MIN; base += 32) {
    const int i = base + lane;
    const bool hit = i < Q - 1 && left[i] + right[i + 1] == best;
    const unsigned m = __ballot_sync(FULL, hit);
    if (m) { split = base + __ffs(m) - 1; ls = left[split]; rs = right[split + 1]; }
  }
  if (split == INT_MIN && lw + right[0] == best) { split = -1; ls = lw; rs = right[0]; }
  if (split == INT_MIN && left[Q - 1] + rw == best) { split = Q - 1; ls = left[Q - 1]; rs = rw; }
  return split == INT_MIN ? make_int4(0, 0, 0, 0) : make_int4(split, ls, rs, 1);
}

/* out[res] = {split row (-1 .. ql-1), upper-left score, lower-right score, 1} or {.., 0} when no row sums to the score */
__global__ void k_align_hirsch(const Prob *probs, int n, const uint8_t *dq, const uint8_t *dt, const uint8_t *code,
                               int nsym, uint8_t *scratch, int4 *out)
{
  const int w = (int)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  const Prob p = probs[w];
  const int Q = p.ql, lw = p.tl / 2, rw = p.tl - lw, best = p.k;
  Scratch sc(scratch + p.scratch, Q, nsym, 1);
  int *left = (int *)((uint8_t *)sc.S + al16((uint64_t)nblocks(Q) * 4));
  int *right = left + Q;
  int dummy0, dummy1;
  if (lw == 0) {  // edlib dereferences a missing column here (T == 1 above the 1 MiB threshold): no alignment
    if (lane == 0) out[p.res] = make_int4(0, 0, 0, 0);
    return;
  }
  build_peq(sc.peq, dq + p.q, Q, false, code, nsym, lane);
  sweep<M_COL>(sc.peq, Q, dt + p.t, lw, false, code, sc.P, sc.M, sc.S, lane, dummy0, dummy1);
  write_column(sc.P, sc.M, sc.S, Q, left, false, lane);
  build_peq(sc.peq, dq + p.q, Q, true, code, nsym, lane);
  sweep<M_COL>(sc.peq, Q, dt + p.t + lw, rw, true, code, sc.P, sc.M, sc.S, lane, dummy0, dummy1);
  write_column(sc.P, sc.M, sc.S, Q, right, true, lane);  // right[i] = NW(query[i..Q), target[lw..T))
  const int4 r = split_row(left, right, Q, lw, rw, best, lane);
  if (lane == 0) out[p.res] = r;
}

/* NW with every column stored, then the traceback (edlib's move preference) from (Q-1, T-1); ops come out in path order */
__global__ void k_align_leaf(const Prob *probs, int n, const uint8_t *dq, const uint8_t *dt, const uint8_t *code, int nsym,
                             uint8_t *scratch, uint8_t *ops, int *out_n)
{
  const int w = (int)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  const Prob p = probs[w];
  const int Q = p.ql, T = p.tl, nb = nblocks(Q);
  Scratch sc(scratch + p.scratch, Q, nsym, (uint64_t)T);
  build_peq(sc.peq, dq + p.q, Q, false, code, nsym, lane);
  int d0, d1;
  sweep<M_STORE>(sc.peq, Q, dt + p.t, T, false, code, sc.P, sc.M, sc.S, lane, d0, d1);
  uint8_t *o = ops + p.out;
  int cnt = 0;
  if (lane == 0) {
    auto val = [&](int i, int j) -> int {
      if (i < 0) return j + 1;
      if (j < 0) return i + 1;
      const size_t x = (size_t)j * nb + (i >> 6);
      const int r = i & 63;
      const uint64_t above = r == 63 ? 0ull : (~0ull << (r + 1));
      return sc.S[x] - __popcll(sc.P[x] & above) + __popcll(sc.M[x] & above);
    };
    int i = Q - 1, j = T - 1;
    while (true) {
      if (i == -1) { for (int x = 0; x <= j; x++) o[cnt++] = 2; break; }
      if (j == -1) { for (int x = 0; x <= i; x++) o[cnt++] = 1; break; }
      const int cur = val(i, j);
      if (val(i - 1, j) + 1 == cur) { o[cnt++] = 1; i--; }
      else if (val(i, j - 1) + 1 == cur) { o[cnt++] = 2; j--; }
      else { o[cnt++] = val(i - 1, j - 1) == cur ? 0 : 3; i--; j--; }
    }
  }
  cnt = __shfl_sync(FULL, cnt, 0);
  __syncwarp();
  for (int x = lane; x < cnt / 2; x += 32) {
    const uint8_t a = o[x];
    o[x] = o[cnt - 1 - x];
    o[cnt - 1 - x] = a;
  }
  if (lane == 0) out_n[p.res] = cnt;
}

/* ---- long sub-problems (max(Q, T) >= MM_ALIGN_BAND_MIN_LEN): a static band, one CTA per sweep ----------------------
 * Band rule (DESIGN.md section 10): with d = i - j and D = Q - T, a cell lies on a path of cost <= k only if
 * |d| + |d - D| <= k, i.e. d in [min(0, D) - w, max(0, D) + w] with w = floor((k - |D|) / 2). Per column the rows of
 * the band form one range whose first and last block are non-decreasing in j and advance by at most one block per
 * column. Blocks outside the range are not computed; scores never underestimate (the first computed block takes the
 * +1 top boundary, a block entering at the bottom starts from the block above plus 64), and a cell whose optimal path
 * stays in the band is exact. The reversed sweep of a Hirschberg node uses the same rule in reversed coordinates. */
constexpr int BAND_BPT = 8;            // blocks a thread keeps in registers over a column tile
constexpr int BAND_INF = 0x3fffffff;   // score of a row outside the band; two of them still sum without overflow

struct Band {
  long long dmin, dmax;
  int Q;
  __host__ __device__ Band(int Q_, int T, int k) : Q(Q_)
  {
    const long long D = (long long)Q_ - T, ad = D < 0 ? -D : D;
    const long long w = k > ad ? (k - ad) / 2 : 0;
    dmin = (D < 0 ? D : 0) - w;
    dmax = (D > 0 ? D : 0) + w;
  }
  __host__ __device__ int first(long long j) const { const long long lo = j + dmin; return lo <= 0 ? 0 : (int)(lo >> 6); }
  __host__ __device__ int last(long long j) const { const long long hi = j + dmax; return (int)((hi < Q - 1 ? hi : Q - 1) >> 6); }
};

__device__ __forceinline__ int myers_block(uint64_t &Pv, uint64_t &Mv, int &sc, uint64_t Eq, int h)
{
  const uint64_t Xv = Eq | Mv;
  if (h < 0) Eq |= 1ull;
  const uint64_t Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
  uint64_t Ph = Mv | ~(Xh | Pv);
  uint64_t Mh = Pv & Xh;
  const int hout = (int)(Ph >> 63) - (int)(Mh >> 63);
  Ph <<= 1;
  Mh <<= 1;
  if (h < 0) Mh |= 1ull;
  else if (h > 0) Ph |= 1ull;
  Pv = Mh | ~(Xv | Ph);
  Mv = Ph & Xv;
  sc += hout;
  return hout;
}

/* score of row 64b + r from a block's P / M words and bottom-row score */
__device__ __forceinline__ int block_row(uint64_t P, uint64_t M, int S, int r)
{
  const uint64_t above = r == 63 ? 0ull : (~0ull << (r + 1));
  return S - __popcll(P & above) + __popcll(M & above);
}

/* Peq of the whole query, built by all warps of the CTA */
__device__ void build_peq_cta(uint64_t *peq, const uint8_t *q, int ql, bool rev, const uint8_t *code, int nsym)
{
  build_peq(peq, q, ql, rev, code, nsym, threadIdx.x & 31, threadIdx.x >> 5, blockDim.x >> 5);
  __syncthreads();
}

/* Banded sweep of a query (its Peq, nb blocks) over ncols target columns (read backwards when trev) by the whole CTA.
 * Block state Ps / Ms / Ss is indexed by absolute block; on return it holds column ncols - 1 for the blocks
 * [bd.first(ncols - 1), bd.last(ncols - 1)].
 *
 * Wavefront: thread t works on column j0 + s - t at step s and passes its horizontal carry (and the bottom score of its
 * last block, for a block entering below it) to thread t + 1 through a shuffle, or shared memory between warps.
 * Ownership is fixed per tile of C = 16 * NT columns: the tile's blocks are the union of its columns' ranges
 * [first(j0), last(j1 - 1)], and thread t owns a fixed contiguous slice of them, kept in registers for the tile. Owning
 * blocks by their position relative to the band instead would break the wavefront's order: when the first block
 * advances, block b at column j - 1 would belong to a thread that reaches column j - 1 after the thread that owns b at
 * column j needs it. The pipeline drains between tiles (NT - 1 idle steps per tile), and the block state goes through
 * global memory only there. A CTA of one warp synchronises with shuffles only. */
__device__ void band_sweep(const uint64_t *peq, int nb, const uint8_t *t, int ncols, bool trev, const uint8_t *code,
                           uint64_t *Ps, uint64_t *Ms, int *Ss, const Band &bd, int *xfer)
{
  const int tid = threadIdx.x, NT = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const bool multi = NT > 32;
  for (int b = bd.first(0) + tid; b <= bd.last(0); b += NT) { Ps[b] = ~0ull; Ms[b] = 0; Ss[b] = 64 * (b + 1); }
  __syncthreads();
  const int C = 16 * NT;
  for (int j0 = 0; j0 < ncols; j0 += C) {
    const int j1 = min(ncols, j0 + C);
    if (j0 > 0 && tid == 0 && bd.last(j0) > bd.last(j0 - 1)) {  // a block entering at the tile's first column
      const int b = bd.last(j0);
      Ps[b] = ~0ull; Ms[b] = 0; Ss[b] = Ss[b - 1] + 64;
    }
    __syncthreads();
    const int u0 = bd.first(j0), u1 = bd.last(j1 - 1);
    const int per = (u1 - u0 + NT) / NT;
    const int s0 = u0 + tid * per, s1 = min(u1 + 1, s0 + per);  // this thread's slice [s0, s1), possibly empty
    uint64_t rP[BAND_BPT], rM[BAND_BPT];
    int rS[BAND_BPT];
    {
      const int f = bd.first(j0), l = bd.last(j0);
#pragma unroll
      for (int i = 0; i < BAND_BPT; i++) {
        const int b = s0 + i;
        const bool on = b < s1 && b >= f && b <= l;
        rP[i] = on ? Ps[b] : 0; rM[i] = on ? Ms[b] : 0; rS[i] = on ? Ss[b] : 0;
      }
    }
    int carry = 0, carry_sc = 0, above = 0;
    const int steps = (j1 - j0) + NT - 1;
    for (int s = 0; s < steps; s++) {
      int hin = __shfl_up_sync(FULL, carry, 1), ain = __shfl_up_sync(FULL, carry_sc, 1);
      if (multi && lane == 0 && warp > 0) {
        const int *x = xfer + (((s + 1) & 1) * 32 + warp - 1) * 2;  // written by the warp above at step s - 1
        hin = x[0]; ain = x[1];
      }
      const int j = j0 + s - tid;
      if (j >= j0 && j < j1) {
        const int f = bd.first(j), l = bd.last(j), lp = j > j0 ? bd.last(j - 1) : l;
        const int b0 = max(s0, f), b1 = min(s1 - 1, l);
        if (b0 <= b1) {
          const uint64_t *pq = peq + (size_t)code[trev ? t[ncols - 1 - j] : t[j]] * nb;
          int h = b0 == f ? 1 : hin;
          // bottom score at column j - 1 of the block above the next one; in a narrow band that block may already have
          // left the band at column j (b < b0) and still holds column j - 1
          int prev = above;
#pragma unroll
          for (int i = 0; i < BAND_BPT; i++) {
            const int b = s0 + i;
            if (b >= b0 && b <= b1) {
              if (b > lp) { rP[i] = ~0ull; rM[i] = 0; rS[i] = prev + 64; }  // enters the band at the bottom
              prev = rS[i];
              h = myers_block(rP[i], rM[i], rS[i], pq[b], h);
              carry_sc = rS[i];
            } else if (b < b0 && b < s1) {
              prev = rS[i];
            }
          }
          if (b0 - 1 >= s0 + BAND_BPT) prev = Ss[b0 - 1];
          for (int b = max(b0, s0 + BAND_BPT); b <= b1; b++) {  // a slice wider than the registers: the rest in memory
            uint64_t Pv = Ps[b], Mv = Ms[b];
            int sc = Ss[b];
            if (b > lp) { Pv = ~0ull; Mv = 0; sc = prev + 64; }
            prev = sc;
            h = myers_block(Pv, Mv, sc, pq[b], h);
            Ps[b] = Pv; Ms[b] = Mv; Ss[b] = sc;
            carry_sc = sc;
          }
          carry = h;
        }
        above = ain;  // bottom score of block s0 - 1 at column j, for a block s0 entering at column j + 1
      }
      if (multi) {
        if (lane == 31) {
          int *x = xfer + ((s & 1) * 32 + warp) * 2;
          x[0] = carry; x[1] = carry_sc;
        }
        __syncthreads();
      } else {
        __syncwarp();
      }
    }
    {
      const int f = bd.first(j1 - 1), l = bd.last(j1 - 1);
#pragma unroll
      for (int i = 0; i < BAND_BPT; i++) {
        const int b = s0 + i;
        if (b < s1 && b >= f && b <= l) { Ps[b] = rP[i]; Ms[b] = rM[i]; Ss[b] = rS[i]; }
      }
    }
    __syncthreads();
  }
}

/* Rule 1' for a long job, one CTA per problem: the banded NW score at (Q-1, T-1) with the band of bound p.k. It is
 * exact when it is <= p.k and an upper bound of the distance otherwise; the host accepts or widens (out[res]). */
__global__ void k_band_nw(const Prob *probs, const uint8_t *dq, const uint8_t *dt, const uint8_t *code, int nsym,
                          uint8_t *scratch, int *out)
{
  __shared__ int xfer[2 * 32 * 2];
  const Prob p = probs[blockIdx.x];
  const int nb = nblocks(p.ql);
  Scratch sc(scratch + p.scratch, p.ql, nsym, 1);
  build_peq_cta(sc.peq, dq + p.q, p.ql, false, code, nsym);
  const Band bd(p.ql, p.tl, p.k);
  band_sweep(sc.peq, nb, dt + p.t, p.tl, false, code, sc.P, sc.M, sc.S, bd, xfer);
  if (threadIdx.x == 0) out[p.res] = block_row(sc.P[nb - 1], sc.M[nb - 1], sc.S[nb - 1], (p.ql - 1) & 63);
}

/* scratch of a long Hirschberg node: two sweep areas (forward, reverse), then left[Q] and right[Q] */
__host__ __device__ inline uint64_t band_node_bytes(int ql, int nsym)
{
  return 2 * scratch_bytes(ql, nsym, 1, 0) + 2 * al16((uint64_t)ql * 4);
}

/* One half of a long Hirschberg node per CTA (blockIdx.x = 2 * node + half): the forward column of the left half or
 * the reverse column of the right half, banded with k = the node's score in the node's own (Q, T). Rows outside the
 * last column's band are BAND_INF. k_band_split takes the split row from the two columns. */
__global__ void k_band_col(const Prob *probs, const uint8_t *dq, const uint8_t *dt, const uint8_t *code, int nsym,
                           uint8_t *scratch)
{
  __shared__ int xfer[2 * 32 * 2];
  const Prob p = probs[blockIdx.x >> 1];
  const bool rev = blockIdx.x & 1;
  const int Q = p.ql, nb = nblocks(Q), lw = p.tl / 2, rw = p.tl - lw;
  if (lw == 0) return;  // no split (k_band_split)
  uint8_t *base = scratch + p.scratch;
  const uint64_t half = scratch_bytes(Q, nsym, 1, 0);
  Scratch sc(base + (rev ? half : 0), Q, nsym, 1);
  int *col = (int *)(base + 2 * half + (rev ? al16((uint64_t)Q * 4) : 0));
  build_peq_cta(sc.peq, dq + p.q, Q, rev, code, nsym);
  const Band bd(Q, p.tl, p.k);
  const int ncols = rev ? rw : lw;
  band_sweep(sc.peq, nb, dt + p.t + (rev ? lw : 0), ncols, rev, code, sc.P, sc.M, sc.S, bd, xfer);
  const int f = bd.first(ncols - 1), l = bd.last(ncols - 1);
  for (int r = threadIdx.x; r < Q; r += blockDim.x) {
    const int b = r >> 6;
    col[rev ? Q - 1 - r : r] = b >= f && b <= l ? block_row(sc.P[b], sc.M[b], sc.S[b], r & 63) : BAND_INF;
  }
}

/* the split of each long node from k_band_col's columns, one warp per node (the ballot scan of k_align_hirsch) */
__global__ void k_band_split(const Prob *probs, int n, int nsym, uint8_t *scratch, int4 *out)
{
  const int w = (int)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  const Prob p = probs[w];
  const int Q = p.ql, lw = p.tl / 2, rw = p.tl - lw;
  if (lw == 0) {  // as k_align_hirsch: a one-column target above the 1 MiB threshold has no alignment
    if (lane == 0) out[p.res] = make_int4(0, 0, 0, 0);
    return;
  }
  const int *left = (const int *)(scratch + p.scratch + 2 * scratch_bytes(Q, nsym, 1, 0));
  const int *right = (const int *)((const uint8_t *)left + al16((uint64_t)Q * 4));
  const int4 r = split_row(left, right, Q, lw, rw, p.k, lane);
  if (lane == 0) out[p.res] = r;
}

/* ---- tag text (mm_align_batch_tags), flat over the ops of a wave of jobs --------------------------------------------
 * The wave's paths lie end to end in one op array (path[x]: the op in bits 0-1, bit 7 on a job's first op). A run is a
 * maximal stretch of one letter inside one job; its text is written by threads balanced over output bytes. */
enum { TAG_CG = 0, TAG_CG_EQX = 1, TAG_CS = 2 };
constexpr uint8_t TAG_FIRST = 0x80;

struct TagLeaf {
  uint64_t src;   // a traced leaf: its ops at ops + src
  uint32_t dst;   // its first op in the wave's paths
  int16_t fill;   // -1: traced; 1 / 2: a leaf with an empty side, all insertions / all deletions
  int16_t first;  // the first leaf of its job
};

struct TagJob {
  uint64_t q, t;   // the job's q_offset / t_offset
  uint32_t op0;    // its first op in the wave's paths
  uint32_t q0, t0; // query / target bases the wave's earlier paths consume
};

/* the letter class of an op: the standard CIGAR folds mismatches into matches */
__device__ __forceinline__ int tag_key(uint8_t p, int kind)
{
  const int op = p & 3;
  return kind == TAG_CG && op == 3 ? 0 : op;
}

__device__ __forceinline__ int tag_digits(uint64_t v)
{
  int d = 1;
  while (v >= 10) { v /= 10; d++; }
  return d;
}

/* digit k (most significant first) of the nd decimal digits of v */
__device__ __forceinline__ char tag_digit(uint64_t v, int nd, int k)
{
  for (int i = nd - 1 - k; i > 0; i--) v /= 10;
  return (char)('0' + v % 10);
}

__device__ __forceinline__ char tag_lower(uint8_t b) { return (char)(b >= 'A' && b <= 'Z' ? b + 32 : b); }

/* last index i in [0, n) with a[i] <= x (a ascending, a[0] <= x) */
template <class T>
__device__ __forceinline__ uint32_t tag_find(const T *a, uint32_t n, uint64_t x)
{
  uint32_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo + 1) >> 1);
    if ((uint64_t)a[mid] <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

/* (1) the wave's leaves compacted into one path per job; a leaf with an empty side is filled here */
__global__ void k_tag_gather(const TagLeaf *leaves, uint32_t n_leaves, const uint8_t *ops, uint32_t n, uint8_t *path)
{
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  uint32_t lo = 0, hi = n_leaves - 1;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo + 1) >> 1);
    if (leaves[mid].dst <= x) lo = mid;
    else hi = mid - 1;
  }
  const TagLeaf l = leaves[lo];
  const uint8_t op = l.fill >= 0 ? (uint8_t)l.fill : ops[l.src + (x - l.dst)];
  path[x] = op | (l.first && x == l.dst ? TAG_FIRST : 0);
}

/* (2) run starts: a job's first op or a change of letter */
__global__ void k_tag_mark(const uint8_t *path, uint32_t n, int kind, uint8_t *mark)
{
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  const uint8_t p = path[x];
  mark[x] = x == 0 || (p & TAG_FIRST) || tag_key(p, kind) != tag_key(path[x - 1], kind);
}

/* (3, 4) per run r < R: its text length and, for cs, the query / target bases it consumes and its job; r = R closes the
 * scans with zeros */
__global__ void k_tag_runs(const uint8_t *path, uint32_t n, const uint32_t *first, uint32_t R, int kind,
                           const TagJob *jobs, uint32_t n_jobs, uint64_t *tlen, uint32_t *qc, uint32_t *tc,
                           uint32_t *rjob)
{
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > R) return;
  if (r == R) {
    tlen[R] = 0;
    if (kind == TAG_CS) { qc[R] = 0; tc[R] = 0; }
    return;
  }
  const uint32_t f = first[r], len = (r + 1 < R ? first[r + 1] : n) - f;
  const int op = path[f] & 3;
  if (kind != TAG_CS) {
    tlen[r] = tag_digits(len) + 1;
    return;
  }
  tlen[r] = op == 0 ? 1 + tag_digits(len) : op == 3 ? 3ull * len : 1ull + len;
  qc[r] = op == 2 ? 0 : len;
  tc[r] = op == 1 ? 0 : len;
  uint32_t lo = 0, hi = n_jobs - 1;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo + 1) >> 1);
    if (jobs[mid].op0 <= f) lo = mid;
    else hi = mid - 1;
  }
  rjob[r] = lo;
}

/* each job's text start: the offset of the run at its first op; j = n_jobs gives the wave's total */
__global__ void k_tag_jobs(const uint32_t *first, uint32_t R, const TagJob *jobs, uint32_t n_jobs, const uint64_t *toff,
                           uint64_t *jtext)
{
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > n_jobs) return;
  jtext[j] = toff[j == n_jobs ? R : tag_find(first, R, jobs[j].op0)];
}

/* (5) one byte of text per thread, its run found by binary search over the run offsets */
__global__ void k_tag_write(const uint8_t *path, uint32_t n, const uint32_t *first, uint32_t R, const uint64_t *toff,
                            uint64_t total, int kind, const uint32_t *qpos, const uint32_t *tpos, const uint32_t *rjob,
                            const TagJob *jobs, const uint8_t *dq, const uint8_t *dt, char *text)
{
  const uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (b >= total) return;
  const uint32_t r = tag_find(toff, R, b);
  const uint64_t k = b - toff[r];
  const uint32_t f = first[r], len = (r + 1 < R ? first[r + 1] : n) - f;
  const int op = path[f] & 3;
  char ch;
  if (kind != TAG_CS) {
    const int nd = tag_digits(len);
    ch = k < (uint64_t)nd ? tag_digit(len, nd, (int)k) : (kind == TAG_CG ? "MIDM" : "=IDX")[op];
  } else if (op == 0) {
    ch = k == 0 ? ':' : tag_digit(len, tag_digits(len), (int)k - 1);
  } else {
    const TagJob &jb = jobs[rjob[r]];
    const uint64_t q = jb.q + (qpos[r] - jb.q0), t = jb.t + (tpos[r] - jb.t0);
    if (op == 3) {
      const uint64_t m = k / 3;
      const int s = (int)(k - 3 * m);
      ch = s == 0 ? '*' : tag_lower(s == 1 ? dt[t + m] : dq[q + m]);
    } else {
      ch = k == 0 ? (op == 1 ? '+' : '-') : tag_lower(op == 1 ? dq[q + k - 1] : dt[t + k - 1]);
    }
  }
  text[b] = ch;
}

thread_local std::string g_create_error;

struct TagBufs {  // device arrays of the formatting pass, grown as needed
  mm_devbuf<TagLeaf> leaves;
  mm_devbuf<TagJob> jobs;
  mm_devbuf<uint8_t> path, mark, tmp;
  mm_devbuf<uint32_t> first, qc, tc, qpos, tpos, rjob;
  mm_devbuf<uint64_t> tlen, toff, jtext;
  mm_devbuf<int64_t> n_runs;
  mm_devbuf<char> text;
};

}  // namespace

struct mm_align_ctx {
  int device = 0;
  uint64_t budget = 0;
  cudaStream_t st = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  std::string err;
  float ms[9] = {0}; /* mm_align_last_stage_ms's 8 slots, then [8] the formatting kernels of mm_align_batch_tags */
  mm_devbuf<uint8_t> q, t, code, scratch, ops;
  mm_devbuf<Prob> probs;
  mm_devbuf<unsigned char> out_a, out_b, out_c, out_n; /* int or int4 results, by stage */
  TagBufs tag;
};

namespace {

struct Failure {
  int code;
};

void ck(mm_align_ctx *c, cudaError_t e, const char *what)
{
  if (e == cudaSuccess) return;
  c->err = std::string(what) + ": " + cudaGetErrorString(e);
  throw Failure{e == cudaErrorMemoryAllocation ? MM_ENOMEM : MM_ECUDA};
}

/* times a stage with events on the context's stream; stage work synchronises itself */
struct StageTimer {
  mm_align_ctx *c;
  int slot;
  StageTimer(mm_align_ctx *c_, int s) : c(c_), slot(s) { ck(c, cudaEventRecord(c->e0, c->st), "event"); }
  ~StageTimer() noexcept(false)
  {
    ck(c, cudaEventRecord(c->e1, c->st), "event");
    ck(c, cudaEventSynchronize(c->e1), "stage");
    float m = 0;
    cudaEventElapsedTime(&m, c->e0, c->e1);
    c->ms[slot] += m;
  }
};

/* Runs kern over probs in waves whose scratch (bytes(p) each) fits the budget. */
template <class Launch, class Bytes>
void run_waves(mm_align_ctx *c, std::vector<Prob> &probs, Bytes bytes, Launch launch)
{
  size_t i = 0;
  while (i < probs.size()) {
    uint64_t used = 0;
    size_t j = i;
    while (j < probs.size()) {
      const uint64_t b = bytes(probs[j]);
      if (j > i && used + b > c->budget) break;
      probs[j].scratch = used;
      used += b;
      j++;
    }
    ck(c, c->scratch.reserve(used), "scratch allocation");
    ck(c, c->probs.reserve(j - i), "problem table allocation");
    ck(c, cudaMemcpyAsync(c->probs.get(), probs.data() + i, (j - i) * sizeof(Prob), cudaMemcpyHostToDevice, c->st), "H2D");
    const int n = (int)(j - i);
    launch(c->probs.get(), n, (n + 3) / 4, 128);
    ck(c, cudaGetLastError(), "kernel launch");
    ck(c, cudaStreamSynchronize(c->st), "kernel");
    i = j;
  }
}

/* the routing rule of the header: a sub-problem's own size decides, so a job's result never depends on its batch */
inline bool is_long(int ql, int tl) { return std::max(ql, tl) >= MM_ALIGN_BAND_MIN_LEN; }

/* threads of the CTA that sweeps a band of bound k: about six blocks per thread, a multiple of 32, 32 to 512. A narrow
 * band (the first passes of the distance schedule) runs as one warp, so it does not pay a CTA barrier per column. */
inline int band_threads(int ql, int tl, int k)
{
  const Band bd(ql, tl, k);
  const long long rows = std::min<long long>(ql, bd.dmax - bd.dmin + 1);
  const long long nt = ((rows / 64 + 2) / 6 + 31) / 32 * 32;
  return (int)std::min<long long>(512, std::max<long long>(32, nt));
}

/* Runs banded problems in launches of one CTA size each (and in waves under the budget); launch(dp, n, threads). */
template <class Launch, class Bytes>
void run_band(mm_align_ctx *c, const std::vector<Prob> &probs, Bytes bytes, Launch launch)
{
  std::vector<int> nt(probs.size());
  for (size_t i = 0; i < probs.size(); i++) nt[i] = band_threads(probs[i].ql, probs[i].tl, probs[i].k);
  std::vector<int> sizes(nt);
  std::sort(sizes.begin(), sizes.end());
  sizes.erase(std::unique(sizes.begin(), sizes.end()), sizes.end());
  for (const int threads : sizes) {
    std::vector<Prob> group;
    for (size_t i = 0; i < probs.size(); i++)
      if (nt[i] == threads) group.push_back(probs[i]);
    run_waves(c, group, bytes, [&](const Prob *dp, int n, int, int) { launch(dp, n, threads); });
  }
}

inline bool is_leaf(int ql, int tl)
{
  if (ql == 0 || tl == 0) return true;
  const long long nb = nblocks(ql);
  return (2 * 8 + 4) * nb * tl + 2 * 4 * (long long)tl < 1024 * 1024;  // edlib.hxx:1156-1158
}

struct Node {
  int job;
  int ql, tl, score;
  uint64_t q, t;
};

/* Validates a batch and gives every distinct byte of it a code (equality is byte identity). */
int check_batch(mm_align_ctx *c, const char *qbases, uint64_t n_q, const char *tbases, uint64_t n_t,
                const mm_align_job *jobs, uint64_t n_jobs, uint8_t code[256], int &nsym)
{
  for (uint64_t j = 0; j < n_jobs; j++) {
    const mm_align_job &b = jobs[j];
    if (b.q_len < 1 || b.t_len < 1 || b.q_offset + (uint64_t)b.q_len > n_q || b.t_offset + (uint64_t)b.t_len > n_t) {
      c->err = "job " + std::to_string(j) + ": empty or out-of-range region";
      return MM_EINVAL;
    }
    if (b.mode != MM_ALIGN_HW && b.mode != MM_ALIGN_NW) {
      c->err = "job " + std::to_string(j) + ": mode " + std::to_string(b.mode) + " is neither MM_ALIGN_HW nor MM_ALIGN_NW";
      return MM_EINVAL;
    }
  }
  nsym = 0;
  if (n_jobs == 0) return MM_OK;
  bool seen[256] = {false};
  for (uint64_t i = 0; i < n_q; i++) seen[(uint8_t)qbases[i]] = true;
  for (uint64_t i = 0; i < n_t; i++) seen[(uint8_t)tbases[i]] = true;
  for (int x = 0; x < 256; x++) code[x] = seen[x] ? (uint8_t)nsym++ : 0;
  if (nsym > 16) {
    c->err = "more than 16 distinct byte values in one batch";
    return MM_EINVAL;
  }
  return MM_OK;
}

/* A batch aligned up to the leaves' traceback (stages 0-4). nodes are the leaves, a job's consecutive and in path
 * order; a leaf with both sides non-empty has its ops in c->ops at off[i] and their count in c->out_n[i]; a leaf with an
 * empty side is all insertions or all deletions and is written by the caller. */
struct Paths {
  std::vector<int> ed, end, start;
  std::vector<Node> nodes;
  std::vector<uint64_t> off;
  std::vector<char> failed;
  int levels = 0;
};

void align_paths(mm_align_ctx *c, const char *qbases, uint64_t n_q, const char *tbases, uint64_t n_t,
                 const mm_align_job *jobs, uint64_t n_jobs, const uint8_t code[256], int nsym, Paths &P)
{
  ck(c, cudaSetDevice(c->device), "cudaSetDevice");
  {
    StageTimer tm(c, 0);
    ck(c, c->q.reserve(n_q), "query allocation");
    ck(c, c->t.reserve(n_t), "target allocation");
    ck(c, c->code.reserve(256), "table allocation");
    ck(c, cudaMemcpyAsync(c->q.get(), qbases, n_q, cudaMemcpyHostToDevice, c->st), "H2D");
    ck(c, cudaMemcpyAsync(c->t.get(), tbases, n_t, cudaMemcpyHostToDevice, c->st), "H2D");
    ck(c, cudaMemcpyAsync(c->code.get(), code, 256, cudaMemcpyHostToDevice, c->st), "H2D");
  }
  const uint8_t *dq = c->q.get(), *dt = c->t.get(), *dc = c->code.get();
  auto sweep_bytes = [nsym](const Prob &p) { return scratch_bytes(p.ql, nsym, 1, 0); };

  // (a) distance and end; HW and NW jobs in launches of their own, long NW jobs banded
  std::vector<int> &ed = P.ed, &end = P.end, &start = P.start;
  ed.assign(n_jobs, 0); end.assign(n_jobs, 0); start.assign(n_jobs, 0);
  std::vector<std::pair<int, int>> band_ed;  // (job, distance) of the long NW jobs
  {
    StageTimer tm(c, 1);
    std::vector<Prob> hw, nw, band;
    for (uint64_t j = 0; j < n_jobs; j++) {
      const mm_align_job &b = jobs[j];
      Prob p{b.q_offset, b.t_offset, b.q_len, b.t_len, b.k, (int)j, 0, 0};
      if (b.mode == MM_ALIGN_NW && is_long(b.q_len, b.t_len)) {
        // k schedule: the first bound leaves 32 diagonals of slack on each side of the length difference
        const long long D = std::abs((long long)b.q_len - b.t_len);
        const long long kmax = b.k < 0 ? std::max(b.q_len, b.t_len) : b.k;
        if (D > kmax) band_ed.push_back({(int)j, -1});  // ed >= |Q - T|
        else { p.k = (int)std::min(kmax, std::max(64LL, D + 64)); band.push_back(p); }
        continue;
      }
      (b.mode == MM_ALIGN_NW ? nw : hw).push_back(p);
    }
    ck(c, c->out_a.reserve(n_jobs * 4), "output allocation");
    ck(c, c->out_b.reserve(n_jobs * 4), "output allocation");
    if (!hw.empty())
      run_waves(c, hw, sweep_bytes, [&](const Prob *dp, int n, int grid, int blk) {
        k_align_hw<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.get(), (int *)c->out_a.get(),
                                            (int *)c->out_b.get());
      });
    if (!nw.empty())
      run_waves(c, nw, sweep_bytes, [&](const Prob *dp, int n, int grid, int blk) {
        k_align_nw<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.get(), (int *)c->out_a.get(),
                                            (int *)c->out_b.get());
      });
    // Banded passes until each long job is decided. A pass's score is exact when it is <= the pass's bound and is the
    // cost of a real path (so >= the distance) otherwise: the next bound is that score or 4x the bound, whichever is
    // smaller, capped at the job's k (k < 0: at max(Q, T), where the band holds every row). A pass at the job's k
    // that stays above it decides -1, as edlib does.
    std::vector<int> v(n_jobs);
    while (!band.empty()) {
      ck(c, c->out_c.reserve(n_jobs * 4), "output allocation");
      run_band(c, band, sweep_bytes, [&](const Prob *dp, int n, int threads) {
        k_band_nw<<<n, threads, 0, c->st>>>(dp, dq, dt, dc, nsym, c->scratch.get(), (int *)c->out_c.get());
      });
      ck(c, cudaMemcpy(v.data(), c->out_c.get(), n_jobs * 4, cudaMemcpyDeviceToHost), "D2H");
      std::vector<Prob> next;
      for (Prob p : band) {
        const mm_align_job &b = jobs[p.res];
        const long long kmax = b.k < 0 ? std::max(b.q_len, b.t_len) : b.k, s = v[p.res];
        if (s <= p.k) band_ed.push_back({p.res, (int)s});
        else if (p.k >= kmax) band_ed.push_back({p.res, -1});
        else { p.k = (int)std::min({kmax, s, 4LL * p.k}); next.push_back(p); }
      }
      band.swap(next);
    }
    ck(c, cudaMemcpyAsync(ed.data(), c->out_a.get(), n_jobs * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
    ck(c, cudaMemcpyAsync(end.data(), c->out_b.get(), n_jobs * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
  }
  for (const auto &x : band_ed) {
    ed[x.first] = x.second;
    end[x.first] = x.second >= 0 ? jobs[x.first].t_len - 1 : -1;
  }
  // (b) start of the HW jobs; end = -1 (the whole query inserted before the target) has start 0, as every NW job has
  {
    StageTimer tm(c, 2);
    std::vector<Prob> probs;
    for (uint64_t j = 0; j < n_jobs; j++)
      if (jobs[j].mode == MM_ALIGN_HW && ed[j] >= 0 && end[j] >= 0)
        probs.push_back(Prob{jobs[j].q_offset, jobs[j].t_offset, jobs[j].q_len, end[j] + 1, 0, (int)j, 0, 0});
    if (!probs.empty()) {
      run_waves(c, probs, sweep_bytes, [&](const Prob *dp, int n, int grid, int blk) {
        k_align_shw<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.get(), (int *)c->out_a.get());
      });
      std::vector<int> s(n_jobs);
      ck(c, cudaMemcpyAsync(s.data(), c->out_a.get(), n_jobs * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
      ck(c, cudaStreamSynchronize(c->st), "D2H");
      for (const Prob &p : probs) start[p.res] = s[p.res];
    }
  }
  // (c) Hirschberg levels; the node list stays in alignment order
  std::vector<Node> &nodes = P.nodes;
  std::vector<char> &failed = P.failed;
  failed.assign(n_jobs, 0);
  for (uint64_t j = 0; j < n_jobs; j++)
    if (ed[j] >= 0)
      nodes.push_back(Node{(int)j, jobs[j].q_len, end[j] - start[j] + 1, ed[j], jobs[j].q_offset,
                           jobs[j].t_offset + (uint64_t)start[j]});
  int &levels = P.levels;
  {
    StageTimer tm(c, 3);
    while (true) {
      std::vector<Prob> probs;
      for (size_t i = 0; i < nodes.size(); i++)
        if (!is_leaf(nodes[i].ql, nodes[i].tl))
          probs.push_back(Prob{nodes[i].q, nodes[i].t, nodes[i].ql, nodes[i].tl, nodes[i].score, (int)probs.size(), 0,
                               i});
      if (probs.empty()) break;
      levels++;
      ck(c, c->out_a.reserve(probs.size() * sizeof(int4)), "output allocation");
      std::vector<Prob> shortp, longp;  // copies: probs keeps the node order for the merge below
      for (const Prob &p : probs) (is_long(p.ql, p.tl) ? longp : shortp).push_back(p);
      if (!shortp.empty())
        run_waves(c, shortp, [nsym](const Prob &p) { return scratch_bytes(p.ql, nsym, 1, (uint64_t)p.ql * 8 + 16); },
                  [&](const Prob *dp, int n, int grid, int blk) {
                    k_align_hirsch<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.get(),
                                                            (int4 *)c->out_a.get());
                  });
      if (!longp.empty())  // both halves of a node as two CTAs, then the split
        run_band(c, longp, [nsym](const Prob &p) { return band_node_bytes(p.ql, nsym); },
                 [&](const Prob *dp, int n, int threads) {
                   k_band_col<<<2 * n, threads, 0, c->st>>>(dp, dq, dt, dc, nsym, c->scratch.get());
                   k_band_split<<<(n + 3) / 4, 128, 0, c->st>>>(dp, n, nsym, c->scratch.get(),
                                                                (int4 *)c->out_a.get());
                 });
      std::vector<int4> sp(probs.size());
      ck(c, cudaMemcpy(sp.data(), c->out_a.get(), sp.size() * sizeof(int4), cudaMemcpyDeviceToHost), "D2H");
      std::vector<Node> next;
      next.reserve(nodes.size() + probs.size());
      size_t pi = 0;
      for (size_t i = 0; i < nodes.size(); i++) {
        const Node &nd = nodes[i];
        if (pi < probs.size() && probs[pi].out == i) {
          const int4 r = sp[pi++];
          if (!r.w) { failed[nd.job] = 1; continue; }
          const int ulh = r.x + 1, lw = nd.tl / 2;
          next.push_back(Node{nd.job, ulh, lw, r.y, nd.q, nd.t});
          next.push_back(Node{nd.job, nd.ql - ulh, nd.tl - lw, r.z, nd.q + (uint64_t)ulh, nd.t + (uint64_t)lw});
        } else {
          next.push_back(nd);
        }
      }
      nodes.swap(next);
    }
  }
  // (d) leaves in waves under the budget; ops of leaf i at [off[i], off[i] + ql + tl)
  std::vector<uint64_t> &off = P.off;
  off.assign(nodes.size() + 1, 0);
  for (size_t i = 0; i < nodes.size(); i++) off[i + 1] = off[i] + (uint64_t)nodes[i].ql + nodes[i].tl;
  {
    StageTimer tm(c, 4);
    std::vector<Prob> probs;
    for (size_t i = 0; i < nodes.size(); i++) {
      const Node &nd = nodes[i];
      if (failed[nd.job]) continue;
      if (nd.ql == 0 || nd.tl == 0) continue;  // all deletions / all insertions (edlib.hxx:1136-1143), filled later
      probs.push_back(Prob{nd.q, nd.t, nd.ql, nd.tl, nd.score, (int)i, 0, off[i]});
    }
    if (!probs.empty()) {
      ck(c, c->ops.reserve(off.back()), "op buffer allocation");
      ck(c, c->out_n.reserve(nodes.size() * 4), "output allocation");
      run_waves(c, probs, [nsym](const Prob &p) { return scratch_bytes(p.ql, nsym, (uint64_t)p.tl, 0); },
                [&](const Prob *dp, int n, int grid, int blk) {
                  k_align_leaf<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.get(),
                                                        c->ops.get(), (int *)c->out_n.get());
                });
    }
  }
}

inline bool traced(const Node &nd) { return nd.ql && nd.tl; }

void cub_run(mm_align_ctx *c, const std::function<cudaError_t(void *, size_t &)> &call)
{
  size_t bytes = 0;
  ck(c, call(nullptr, bytes), "cub");
  ck(c, c->tag.tmp.reserve(bytes + 16), "cub temporary allocation");
  ck(c, call(c->tag.tmp.get(), bytes), "cub");
}

inline unsigned grid256(uint64_t n) { return (unsigned)((n + 255) / 256); }

/* One formatting pass over a wave's paths (c->tag.path, n ops, nj jobs): jtext[w] = the text offset of wave job w
 * (jtext[nj] = the pass's total). The text is written, to host[0, total), only when it fits in room bytes. */
void format_pass(mm_align_ctx *c, uint32_t n, uint32_t nj, int kind, char *host, uint64_t room,
                 std::vector<uint64_t> &jtext)
{
  TagBufs &g = c->tag;
  int64_t R = 0;
  {
    StageTimer tm(c, 8);
    k_tag_mark<<<grid256(n), 256, 0, c->st>>>(g.path.get(), n, kind, g.mark.get());
    ck(c, cudaGetLastError(), "kernel launch");
    const cub::CountingInputIterator<uint32_t> idx(0);
    cub_run(c, [&](void *t, size_t &bytes) {
      return cub::DeviceSelect::Flagged(t, bytes, idx, g.mark.get(), g.first.get(), g.n_runs.get(), (int64_t)n, c->st);
    });
    ck(c, cudaMemcpyAsync(&R, g.n_runs.get(), 8, cudaMemcpyDeviceToHost, c->st), "D2H");
    ck(c, cudaStreamSynchronize(c->st), "run starts");
    const uint32_t r = (uint32_t)R;
    k_tag_runs<<<grid256(r + 1ull), 256, 0, c->st>>>(g.path.get(), n, g.first.get(), r, kind, g.jobs.get(), nj,
                                                    g.tlen.get(), g.qc.get(), g.tc.get(), g.rjob.get());
    ck(c, cudaGetLastError(), "kernel launch");
    cub_run(c, [&](void *t, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(t, bytes, g.tlen.get(), g.toff.get(), (int64_t)r + 1, c->st);
    });
    if (kind == TAG_CS) {
      cub_run(c, [&](void *t, size_t &bytes) {
        return cub::DeviceScan::ExclusiveSum(t, bytes, g.qc.get(), g.qpos.get(), (int64_t)r + 1, c->st);
      });
      cub_run(c, [&](void *t, size_t &bytes) {
        return cub::DeviceScan::ExclusiveSum(t, bytes, g.tc.get(), g.tpos.get(), (int64_t)r + 1, c->st);
      });
    }
    k_tag_jobs<<<grid256(nj + 1ull), 256, 0, c->st>>>(g.first.get(), r, g.jobs.get(), nj, g.toff.get(), g.jtext.get());
    ck(c, cudaGetLastError(), "kernel launch");
    jtext.resize(nj + 1);
    ck(c, cudaMemcpyAsync(jtext.data(), g.jtext.get(), (nj + 1) * 8, cudaMemcpyDeviceToHost, c->st), "D2H");
    ck(c, cudaStreamSynchronize(c->st), "run text offsets");
    if (jtext[nj] > room) return;
    const uint64_t total = jtext[nj];
    ck(c, g.text.reserve(total), "text allocation");
    k_tag_write<<<grid256(total), 256, 0, c->st>>>(g.path.get(), n, g.first.get(), r, g.toff.get(), total, kind,
                                                  g.qpos.get(), g.tpos.get(), g.rjob.get(), g.jobs.get(), c->q.get(),
                                                  c->t.get(), g.text.get());
    ck(c, cudaGetLastError(), "kernel launch");
  }
  StageTimer tm(c, 5);
  ck(c, cudaMemcpyAsync(host, g.text.get(), jtext[nj], cudaMemcpyDeviceToHost, c->st), "D2H");
}

/* mm_align_batch_tags after align_paths: the traced leaves' lengths come back, then the paths are formatted in waves of
 * whole jobs of at most `cap` ops (a longer job is a wave of its own), which bounds the pass's device arrays. */
uint64_t format_tags(mm_align_ctx *c, const mm_align_job *jobs, uint64_t n_jobs, uint32_t flags, const Paths &P,
                     mm_align_tag_result *results, char *text, uint64_t text_cap)
{
  const std::vector<Node> &nodes = P.nodes;
  std::vector<int> dn(nodes.size(), 0);
  bool any = false;
  for (const Node &nd : nodes) any |= !P.failed[nd.job] && traced(nd);
  if (any) {
    StageTimer tm(c, 5);
    ck(c, cudaMemcpyAsync(dn.data(), c->out_n.get(), nodes.size() * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
  }
  std::vector<uint64_t> len(n_jobs, 0);
  for (size_t i = 0; i < nodes.size(); i++)
    if (!P.failed[nodes[i].job]) len[nodes[i].job] += traced(nodes[i]) ? dn[i] : nodes[i].ql + nodes[i].tl;
  for (uint64_t j = 0; j < n_jobs; j++)
    results[j] = mm_align_tag_result{P.ed[j], P.failed[j] ? 0 : (int32_t)len[j], 0, 0, 0, 0};

  // about 48 bytes of device arrays per op: a wave takes about a quarter of the scratch budget
  const uint64_t cap = std::min<uint64_t>(std::max<uint64_t>(c->budget / (4 * 48), 1u << 20), 1u << 30);
  struct Wave {
    std::vector<TagJob> jobs;
    std::vector<TagLeaf> leaves;
    std::vector<uint64_t> ids;
    uint64_t n = 0;
  };
  std::vector<Wave> waves;
  uint64_t max_n = 0, max_leaves = 0, max_jobs = 0;
  size_t ni = 0;
  for (uint64_t j = 0; j < n_jobs; j++) {
    if (P.failed[j] || len[j] == 0) continue;
    if (waves.empty() || waves.back().n + len[j] > cap) waves.emplace_back();
    Wave &w = waves.back();
    uint64_t q0 = 0, t0 = 0;
    if (!w.ids.empty()) {
      const mm_align_job &prev = jobs[w.ids.back()];
      q0 = w.jobs.back().q0 + prev.q_len;
      t0 = w.jobs.back().t0 + prev.t_len;
    }
    w.jobs.push_back(TagJob{jobs[j].q_offset, jobs[j].t_offset, (uint32_t)w.n, (uint32_t)q0, (uint32_t)t0});
    w.ids.push_back(j);
    while (nodes[ni].job < (int)j) ni++;
    for (bool first = true; ni < nodes.size() && nodes[ni].job == (int)j; ni++, first = false) {
      const Node &nd = nodes[ni];
      w.leaves.push_back(TagLeaf{P.off[ni], (uint32_t)w.n, (int16_t)(traced(nd) ? -1 : nd.ql == 0 ? 2 : 1), first});
      w.n += traced(nd) ? dn[ni] : nd.ql + nd.tl;
    }
    max_n = std::max(max_n, w.n);
    max_leaves = std::max<uint64_t>(max_leaves, w.leaves.size());
    max_jobs = std::max<uint64_t>(max_jobs, w.jobs.size());
  }
  if (waves.empty()) return 0;

  // Everything is sized for the largest wave before the first launch: an array that grows frees its old one, and
  // cudaFree waits for the whole device, including the mapping kernels that run beside the aligner.
  const int kinds[2] = {flags & MM_ALIGN_TAG_EQX ? TAG_CG_EQX : TAG_CG, TAG_CS};
  const int passes = flags & MM_ALIGN_TAG_CS ? 2 : 1;
  TagBufs &g = c->tag;
  ck(c, g.leaves.reserve(max_leaves), "leaf table allocation");
  ck(c, g.jobs.reserve(max_jobs), "job table allocation");
  ck(c, g.jtext.reserve(max_jobs + 1), "job text allocation");
  ck(c, g.path.reserve(max_n), "path allocation");
  ck(c, g.mark.reserve(max_n), "run allocation");
  ck(c, g.first.reserve(max_n), "run allocation");
  ck(c, g.tlen.reserve(max_n + 1), "run allocation");
  ck(c, g.toff.reserve(max_n + 1), "run allocation");
  ck(c, g.n_runs.reserve(1), "run allocation");
  ck(c, g.text.reserve(max_n * (passes == 2 ? 3 : 2)), "text allocation");  // 2 bytes of cg, 3 of cs per op at most
  if (passes == 2)
    for (mm_devbuf<uint32_t> *b : {&g.qc, &g.tc, &g.qpos, &g.tpos, &g.rjob})
      ck(c, b->reserve(max_n + 1), "run allocation");
  {
    size_t b0 = 0, b1 = 0, b2 = 0;
    const cub::CountingInputIterator<uint32_t> idx(0);
    ck(c, cub::DeviceSelect::Flagged(nullptr, b0, idx, g.mark.get(), g.first.get(), g.n_runs.get(), (int64_t)max_n,
                                     c->st), "cub");
    ck(c, cub::DeviceScan::ExclusiveSum(nullptr, b1, g.tlen.get(), g.toff.get(), (int64_t)max_n + 1, c->st), "cub");
    ck(c, cub::DeviceScan::ExclusiveSum(nullptr, b2, g.qc.get(), g.qpos.get(), (int64_t)max_n + 1, c->st), "cub");
    ck(c, g.tmp.reserve(std::max({b0, b1, b2}) + 16), "cub temporary allocation");
  }
  uint64_t pos = 0;
  for (const Wave &w : waves) {
    const uint32_t nj = (uint32_t)w.jobs.size();
    ck(c, cudaMemcpyAsync(g.leaves.get(), w.leaves.data(), w.leaves.size() * sizeof(TagLeaf), cudaMemcpyHostToDevice,
                          c->st), "H2D");
    ck(c, cudaMemcpyAsync(g.jobs.get(), w.jobs.data(), nj * sizeof(TagJob), cudaMemcpyHostToDevice, c->st), "H2D");
    {
      StageTimer tm(c, 8);
      k_tag_gather<<<grid256(w.n), 256, 0, c->st>>>(g.leaves.get(), (uint32_t)w.leaves.size(), c->ops.get(),
                                                    (uint32_t)w.n, g.path.get());
      ck(c, cudaGetLastError(), "kernel launch");
    }
    for (int k = 0; k < passes; k++) {
      std::vector<uint64_t> jt;
      // past the caller's buffer only the size is still needed
      format_pass(c, (uint32_t)w.n, nj, kinds[k], text + std::min(pos, text_cap), pos <= text_cap ? text_cap - pos : 0,
                  jt);
      for (uint32_t x = 0; x < nj; x++) {
        mm_align_tag_result &r = results[w.ids[x]];
        (k == 0 ? r.cg_offset : r.cs_offset) = pos + jt[x];
        (k == 0 ? r.cg_len : r.cs_len) = jt[x + 1] - jt[x];
      }
      pos += jt[nj];
    }
  }
  return pos;
}

}  // namespace

extern "C" {

int mm_align_ctx_create(int device, uint64_t scratch_bytes, mm_align_ctx **out)
{
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
    g_create_error = "no CUDA device " + std::to_string(device);
    return MM_ENODEVICE;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
    g_create_error = "device " + std::to_string(device) + " is not compute capability 9.0 (sm_90a)";
    return MM_ENODEVICE;
  }
  auto *c = new mm_align_ctx();
  c->device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreate(&c->e0) != cudaSuccess || cudaEventCreate(&c->e1) != cudaSuccess) {
    g_create_error = "CUDA context / stream creation failed";
    delete c;
    return MM_ECUDA;
  }
  if (scratch_bytes == 0) {
    size_t fr = 0, tot = 0;
    cudaMemGetInfo(&fr, &tot);
    scratch_bytes = std::min<uint64_t>(fr / 2, 8ull << 30);
  }
  c->budget = std::max<uint64_t>(scratch_bytes, 4ull << 20);
  *out = c;
  return MM_OK;
}

int mm_align_ctx_destroy(mm_align_ctx *ctx)
{
  if (!ctx) return MM_OK;
  cudaSetDevice(ctx->device);
  if (ctx->st) cudaStreamSynchronize(ctx->st);
  if (ctx->e0) cudaEventDestroy(ctx->e0);
  if (ctx->e1) cudaEventDestroy(ctx->e1);
  if (ctx->st) cudaStreamDestroy(ctx->st);
  delete ctx;
  return MM_OK;
}

const char *mm_align_last_error(const mm_align_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int mm_align_last_stage_ms(const mm_align_ctx *ctx, float ms[8])
{
  if (!ctx || !ms) return MM_EINVAL;
  std::memcpy(ms, ctx->ms, 8 * sizeof(float));
  return MM_OK;
}

int mm_align_batch(mm_align_ctx *c, const char *qbases, uint64_t n_q, const char *tbases, uint64_t n_t,
                   const mm_align_job *jobs, uint64_t n_jobs, mm_align_result *results, uint8_t *ops, uint64_t ops_cap,
                   uint64_t *n_ops)
{
  if (!c || (n_jobs && (!jobs || !results || !n_ops))) return MM_EINVAL;
  const auto h0 = std::chrono::steady_clock::now();
  std::fill(c->ms, c->ms + 8, 0.f);
  *n_ops = 0;
  uint8_t code[256];
  int nsym = 0;
  if (const int rc = check_batch(c, qbases, n_q, tbases, n_t, jobs, n_jobs, code, nsym)) return rc;
  if (n_jobs == 0) return MM_OK;
  try {
    Paths P;
    align_paths(c, qbases, n_q, tbases, n_t, jobs, n_jobs, code, nsym, P);
    const std::vector<Node> &nodes = P.nodes;
    const std::vector<uint64_t> &off = P.off;
    const std::vector<char> &failed = P.failed;
    const std::vector<int> &ed = P.ed, &start = P.start, &end = P.end;
    std::vector<uint8_t> leaf_ops(off.back());
    std::vector<int> leaf_n(nodes.size(), 0);
    for (size_t i = 0; i < nodes.size(); i++) {
      const Node &nd = nodes[i];
      if (failed[nd.job] || traced(nd)) continue;
      std::fill(leaf_ops.begin() + off[i], leaf_ops.begin() + off[i] + nd.ql + nd.tl, nd.ql == 0 ? 2 : 1);
      leaf_n[i] = nd.ql + nd.tl;
    }
    {
      StageTimer tm(c, 5);
      bool any = false;
      for (size_t i = 0; i < nodes.size(); i++) any |= !failed[nodes[i].job] && nodes[i].ql && nodes[i].tl;
      if (any) {
        std::vector<int> dn(nodes.size());
        ck(c, cudaMemcpyAsync(dn.data(), c->out_n.get(), nodes.size() * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
        std::vector<uint8_t> dops(off.back());
        ck(c, cudaMemcpyAsync(dops.data(), c->ops.get(), off.back(), cudaMemcpyDeviceToHost, c->st), "D2H");
        ck(c, cudaStreamSynchronize(c->st), "D2H");
        for (size_t i = 0; i < nodes.size(); i++)
          if (!failed[nodes[i].job] && nodes[i].ql && nodes[i].tl) {
            leaf_n[i] = dn[i];
            std::memcpy(leaf_ops.data() + off[i], dops.data() + off[i], dn[i]);
          }
      }
    }
    // results: a job's leaves are consecutive in the list and in path order
    std::vector<uint64_t> len(n_jobs, 0);
    for (size_t i = 0; i < nodes.size(); i++)
      if (!failed[nodes[i].job]) len[nodes[i].job] += leaf_n[i];
    uint64_t total = 0;
    for (uint64_t j = 0; j < n_jobs; j++) {
      results[j].ed = ed[j];
      results[j].start = ed[j] >= 0 ? start[j] : -1;
      results[j].end = ed[j] >= 0 ? end[j] : -1;
      results[j].alignment_length = failed[j] ? 0 : (int)len[j];
      results[j].ops_offset = total;
      total += failed[j] ? 0 : len[j];
    }
    *n_ops = total;
    if (total > ops_cap) {
      c->err = "op buffer too small";
      return MM_ECAPACITY;
    }
    for (size_t i = 0; i < nodes.size(); i++) {
      const Node &nd = nodes[i];
      if (failed[nd.job]) continue;
      mm_align_result &r = results[nd.job];
      std::memcpy(ops + r.ops_offset, leaf_ops.data() + off[i], leaf_n[i]);
      r.ops_offset += leaf_n[i];
    }
    for (uint64_t j = 0; j < n_jobs; j++) results[j].ops_offset -= failed[j] ? 0 : len[j];
    c->ms[7] = (float)P.levels;
  } catch (const Failure &f) {
    return f.code;
  }
  c->ms[6] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - h0).count();
  return MM_OK;
}

int mm_align_batch_tags(mm_align_ctx *c, const char *qbases, uint64_t n_q, const char *tbases, uint64_t n_t,
                        const mm_align_job *jobs, uint64_t n_jobs, uint32_t flags, mm_align_tag_result *results,
                        char *text, uint64_t text_cap, uint64_t *n_text)
{
  if (!c || (n_jobs && (!jobs || !results || !n_text)) || (text_cap && !text)) return MM_EINVAL;
  const auto h0 = std::chrono::steady_clock::now();
  std::fill(c->ms, c->ms + 9, 0.f);
  if (n_text) *n_text = 0;
  if (flags & ~(uint32_t)(MM_ALIGN_TAG_EQX | MM_ALIGN_TAG_CS)) {
    c->err = "flags " + std::to_string(flags) + " hold bits other than MM_ALIGN_TAG_EQX and MM_ALIGN_TAG_CS";
    return MM_EINVAL;
  }
  uint8_t code[256];
  int nsym = 0;
  if (const int rc = check_batch(c, qbases, n_q, tbases, n_t, jobs, n_jobs, code, nsym)) return rc;
  for (uint64_t j = 0; j < n_jobs; j++)
    if (jobs[j].mode != MM_ALIGN_NW) {
      c->err = "job " + std::to_string(j) + ": mm_align_batch_tags takes MM_ALIGN_NW jobs only";
      return MM_EINVAL;
    }
  if (n_jobs == 0) return MM_OK;
  try {
    Paths P;
    align_paths(c, qbases, n_q, tbases, n_t, jobs, n_jobs, code, nsym, P);
    *n_text = format_tags(c, jobs, n_jobs, flags, P, results, text, text_cap);
    c->ms[7] = (float)P.levels;
    if (*n_text > text_cap) {
      c->err = "text buffer too small";
      return MM_ECAPACITY;
    }
  } catch (const Failure &f) {
    return f.code;
  }
  c->ms[6] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - h0).count();
  return MM_OK;
}

int mm_align_last_tag_ms(const mm_align_ctx *ctx, float *ms)
{
  if (!ctx || !ms) return MM_EINVAL;
  *ms = ctx->ms[8];
  return MM_OK;
}

}  // extern "C"
