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
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mashmap_b200_align.h"

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

/* Peq[s * nb + b]: bit i set when query row 64b + i holds symbol s; rows past the query (padding) match everything. */
__device__ void build_peq(uint64_t *peq, const uint8_t *q, int ql, bool rev, const uint8_t *code, int nsym, int lane)
{
  const int nb = nblocks(ql);
  for (int b = 0; b < nb; b++) {
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
__host__ inline uint64_t scratch_bytes(int ql, int nsym, uint64_t cols, uint64_t extra)
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
  int split = INT_MIN, ls = 0, rs = 0;
  for (int base = 0; base < Q - 1 && split == INT_MIN; base += 32) {
    const int i = base + lane;
    const bool hit = i < Q - 1 && left[i] + right[i + 1] == best;
    const unsigned m = __ballot_sync(FULL, hit);
    if (m) { split = base + __ffs(m) - 1; ls = left[split]; rs = right[split + 1]; }
  }
  if (split == INT_MIN && lw + right[0] == best) { split = -1; ls = lw; rs = right[0]; }
  if (split == INT_MIN && left[Q - 1] + rw == best) { split = Q - 1; ls = left[Q - 1]; rs = rw; }
  if (lane == 0) out[p.res] = split == INT_MIN ? make_int4(0, 0, 0, 0) : make_int4(split, ls, rs, 1);
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

struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n)
  {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(n, 256));
    if (e == cudaSuccess) cap = std::max<size_t>(n, 256);
    return e;
  }
  template <class T> T *as() const { return (T *)p; }
  ~DevBuf() { if (p) cudaFree(p); }
};

thread_local std::string g_create_error;

}  // namespace

struct mm_align_ctx {
  int device = 0;
  uint64_t budget = 0;
  cudaStream_t st = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  std::string err;
  float ms[8] = {0};
  DevBuf q, t, code, probs, scratch, out_a, out_b, ops, out_n;
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
    ck(c, c->scratch.ensure(used), "scratch allocation");
    ck(c, c->probs.ensure((j - i) * sizeof(Prob)), "problem table allocation");
    ck(c, cudaMemcpyAsync(c->probs.p, probs.data() + i, (j - i) * sizeof(Prob), cudaMemcpyHostToDevice, c->st), "H2D");
    const int n = (int)(j - i);
    launch(c->probs.as<Prob>(), n, (n + 3) / 4, 128);
    ck(c, cudaGetLastError(), "kernel launch");
    ck(c, cudaStreamSynchronize(c->st), "kernel");
    i = j;
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
  std::memcpy(ms, ctx->ms, sizeof(ctx->ms));
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
  if (n_jobs == 0) return MM_OK;
  // symbols: every distinct byte of the batch gets a code (equality is byte identity)
  uint8_t code[256];
  bool seen[256] = {false};
  for (uint64_t i = 0; i < n_q; i++) seen[(uint8_t)qbases[i]] = true;
  for (uint64_t i = 0; i < n_t; i++) seen[(uint8_t)tbases[i]] = true;
  int nsym = 0;
  for (int x = 0; x < 256; x++) code[x] = seen[x] ? (uint8_t)nsym++ : 0;
  if (nsym > 16) {
    c->err = "more than 16 distinct byte values in one batch";
    return MM_EINVAL;
  }
  try {
    ck(c, cudaSetDevice(c->device), "cudaSetDevice");
    {
      StageTimer tm(c, 0);
      ck(c, c->q.ensure(n_q), "query allocation");
      ck(c, c->t.ensure(n_t), "target allocation");
      ck(c, c->code.ensure(256), "table allocation");
      ck(c, cudaMemcpyAsync(c->q.p, qbases, n_q, cudaMemcpyHostToDevice, c->st), "H2D");
      ck(c, cudaMemcpyAsync(c->t.p, tbases, n_t, cudaMemcpyHostToDevice, c->st), "H2D");
      ck(c, cudaMemcpyAsync(c->code.p, code, 256, cudaMemcpyHostToDevice, c->st), "H2D");
    }
    const uint8_t *dq = c->q.as<uint8_t>(), *dt = c->t.as<uint8_t>(), *dc = c->code.as<uint8_t>();
    auto sweep_bytes = [nsym](const Prob &p) { return scratch_bytes(p.ql, nsym, 1, 0); };

    // (a) distance and end; HW and NW jobs in launches of their own
    std::vector<int> ed(n_jobs), end(n_jobs), start(n_jobs, 0);
    {
      StageTimer tm(c, 1);
      std::vector<Prob> hw, nw;
      for (uint64_t j = 0; j < n_jobs; j++)
        (jobs[j].mode == MM_ALIGN_NW ? nw : hw)
            .push_back(Prob{jobs[j].q_offset, jobs[j].t_offset, jobs[j].q_len, jobs[j].t_len, jobs[j].k, (int)j, 0, 0});
      ck(c, c->out_a.ensure(n_jobs * 4), "output allocation");
      ck(c, c->out_b.ensure(n_jobs * 4), "output allocation");
      if (!hw.empty())
        run_waves(c, hw, sweep_bytes, [&](const Prob *dp, int n, int grid, int blk) {
          k_align_hw<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.as<uint8_t>(), c->out_a.as<int>(),
                                              c->out_b.as<int>());
        });
      if (!nw.empty())
        run_waves(c, nw, sweep_bytes, [&](const Prob *dp, int n, int grid, int blk) {
          k_align_nw<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.as<uint8_t>(), c->out_a.as<int>(),
                                              c->out_b.as<int>());
        });
      ck(c, cudaMemcpyAsync(ed.data(), c->out_a.p, n_jobs * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
      ck(c, cudaMemcpyAsync(end.data(), c->out_b.p, n_jobs * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
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
          k_align_shw<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.as<uint8_t>(), c->out_a.as<int>());
        });
        std::vector<int> s(n_jobs);
        ck(c, cudaMemcpyAsync(s.data(), c->out_a.p, n_jobs * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
        ck(c, cudaStreamSynchronize(c->st), "D2H");
        for (const Prob &p : probs) start[p.res] = s[p.res];
      }
    }
    // (c) Hirschberg levels; the node list stays in alignment order
    std::vector<Node> nodes;
    std::vector<char> failed(n_jobs, 0);
    for (uint64_t j = 0; j < n_jobs; j++)
      if (ed[j] >= 0)
        nodes.push_back(Node{(int)j, jobs[j].q_len, end[j] - start[j] + 1, ed[j], jobs[j].q_offset,
                             jobs[j].t_offset + (uint64_t)start[j]});
    int levels = 0;
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
        ck(c, c->out_a.ensure(probs.size() * sizeof(int4)), "output allocation");
        run_waves(c, probs, [nsym](const Prob &p) { return scratch_bytes(p.ql, nsym, 1, (uint64_t)p.ql * 8 + 16); },
                  [&](const Prob *dp, int n, int grid, int blk) {
                    k_align_hirsch<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.as<uint8_t>(),
                                                            c->out_a.as<int4>());
                  });
        std::vector<int4> sp(probs.size());
        ck(c, cudaMemcpy(sp.data(), c->out_a.p, sp.size() * sizeof(int4), cudaMemcpyDeviceToHost), "D2H");
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
    std::vector<uint64_t> off(nodes.size() + 1, 0);
    for (size_t i = 0; i < nodes.size(); i++) off[i + 1] = off[i] + (uint64_t)nodes[i].ql + nodes[i].tl;
    std::vector<uint8_t> leaf_ops(off.back());
    std::vector<int> leaf_n(nodes.size(), 0);
    {
      StageTimer tm(c, 4);
      std::vector<Prob> probs;
      for (size_t i = 0; i < nodes.size(); i++) {
        const Node &nd = nodes[i];
        if (failed[nd.job]) continue;
        if (nd.ql == 0 || nd.tl == 0) {  // all deletions / all insertions (edlib.hxx:1136-1143)
          std::fill(leaf_ops.begin() + off[i], leaf_ops.begin() + off[i] + nd.ql + nd.tl, nd.ql == 0 ? 2 : 1);
          leaf_n[i] = nd.ql + nd.tl;
          continue;
        }
        probs.push_back(Prob{nd.q, nd.t, nd.ql, nd.tl, nd.score, (int)i, 0, off[i]});
      }
      if (!probs.empty()) {
        ck(c, c->ops.ensure(off.back()), "op buffer allocation");
        ck(c, c->out_n.ensure(nodes.size() * 4), "output allocation");
        run_waves(c, probs, [nsym](const Prob &p) { return scratch_bytes(p.ql, nsym, (uint64_t)p.tl, 0); },
                  [&](const Prob *dp, int n, int grid, int blk) {
                    k_align_leaf<<<grid, blk, 0, c->st>>>(dp, n, dq, dt, dc, nsym, c->scratch.as<uint8_t>(),
                                                          c->ops.as<uint8_t>(), c->out_n.as<int>());
                  });
      }
    }
    {
      StageTimer tm(c, 5);
      bool any = false;
      for (size_t i = 0; i < nodes.size(); i++) any |= !failed[nodes[i].job] && nodes[i].ql && nodes[i].tl;
      if (any) {
        std::vector<int> dn(nodes.size());
        ck(c, cudaMemcpyAsync(dn.data(), c->out_n.p, nodes.size() * 4, cudaMemcpyDeviceToHost, c->st), "D2H");
        std::vector<uint8_t> dops(off.back());
        ck(c, cudaMemcpyAsync(dops.data(), c->ops.p, off.back(), cudaMemcpyDeviceToHost, c->st), "D2H");
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
    c->ms[7] = (float)levels;
  } catch (const Failure &f) {
    return f.code;
  }
  c->ms[6] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - h0).count();
  return MM_OK;
}

}  // extern "C"
