/*
 * mm_sketch.cu -- K0 (base packing) and K1: bottom-s MinHash sketch of every query segment.
 *
 * Replaces CommonFunc::sketchSequence (reference src/map/include/commonFunc.hpp:182-288) as
 * called from Map::getSeedHits (computeMap.hpp:817-843), i.e. rows a1-a3 of SURVEY 8(a):
 *   normalise bases (commonFunc.hpp:97-107), hash every k-mer and its reverse complement with
 *   MurmurHash3_x64_128 (commonFunc.hpp:225-237), keep k-mers without N whose two hashes differ
 *   (:234), canonical = min (:237), strand vote = +1 if fwd < rev else -1 (:240), and output the
 *   s smallest DISTINCT canonical hashes with first position, last position and the sign of the
 *   vote sum (:242-286), ascending by hash.
 * sketchSequence is a pure set function (SURVEY A.4: the heap top only decreases once full, so
 * every occurrence of a surviving hash is seen), so any selection that yields that set is
 * bit-exact. This file does it without a heap:
 *
 *   K0 k_pack_bases: makeUpperCaseAndValidDNA (commonFunc.hpp:97-107) as a format change -- every base becomes one
 *     nibble: 2-bit code (A=0 C=1 T=2 G=3: bits 1-2 of the upper-cased letter) | 8 for anything that is not ACGT.
 *     HBM-bound (1 B read + 0.5 B written per base). Hosts that pack while they parse (skch::BatchMapper) upload the
 *     nibbles directly and skip it.
 *   K1 k_sketch: one CTA per segment (persistent grid); the segment's nibbles are staged HBM -> shared memory with a
 *     1-D TMA bulk copy (cp.async.bulk + mbarrier, double buffered across segments). Each thread owns a contiguous run of
 *     k-mer positions, four per step: the ASCII bytes of the forward k-mers and of their reverse complements are
 *     rebuilt in registers from the nibbles with byte permutes (PRMT: a 4-entry lookup per nibble, then one permute per
 *     32-bit window word per position), so no base is decoded one at a time. Both Murmur3 evaluations run on those
 *     words (INT-ALU bound: ~10 64-bit multiplies each). A position whose smaller hash has a leading word <= T's
 *     (T ~ c*s/n * 2^64) is kept, raw, in a per-thread list in shared memory; after the run every thread inserts its own
 *     list into a shared-memory open-addressing table keyed by hash (atomicCAS) that accumulates first position / last
 *     position / vote sum (atomicMin / atomicMax / atomicAdd) -- de-duplication before any sorting. If fewer than s
 *     distinct hashes survived although larger ones exist, or the table overflowed, T is raised / lowered / bisected and
 *     the pass is redone (rare; always terminates because distinct-count(T) grows by at most one per unit of T). The
 *     <= C survivors are ordered with a 256-bucket counting sort on the leading bits plus in-bucket ranking, and the
 *     first s are written out. Where the batch has an index (sk_val set), every hash written is also looked up in the
 *     index's table (K2's first step, whose DRAM latency here overlaps the other CTAs' hashing).
 *   A thread whose stretch of the segment contains an N (nibble bit 3) takes the same loop with the run-length test
 *   of commonFunc.hpp:207-223 compiled in; all others skip it.
 */
#include <cub/cub.cuh>

#include "mm_internal.h"

namespace {

#ifndef MM_SK_THREADS
#define MM_SK_THREADS 128
#endif
constexpr int SK_THREADS = MM_SK_THREADS;
#ifndef MM_SK_MINB
#define MM_SK_MINB 7 /* minimum resident CTAs per SM the fast kernel is compiled for (register budget = 65536 / (MINB * threads)) */
#endif
constexpr int SK_BUCKETS = 256;
constexpr uint64_t SK_EMPTY = ~0ULL;
constexpr uint32_t SK_POOL_FWD = 0x47544341u;  /* ASCII by code: A C T G */
constexpr uint32_t SK_POOL_COMP = 0x43414754u; /* ASCII of the complement by code: T G A C */

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
/* 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP) */
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "MM_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra MM_DONE;\n"
      "bra MM_WAIT;\n"
      "MM_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel)
{
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}

/* ---------------------------------------------------------------------------------------------------------------
 * K0: ASCII -> nibbles. 16 bases per thread and step (one 16-byte load, one 8-byte store).
 * ------------------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint32_t pack4(uint32_t w)
{ /* 4 ASCII bytes -> 4 nibbles in the low 16 bits (base 0 in bits 0-3) */
  const uint32_t x = w & 0xDFDFDFDFu;                 /* a-z -> A-Z (commonFunc.hpp:100-101) */
  uint32_t code = (x >> 1) & 0x03030303u;             /* A=0 C=1 T=2 G=3 */
  const uint32_t t = code | (code >> 4);              /* byte0 = c0|c1<<4, byte2 = c2|c3<<4 */
  const uint32_t sel = prmt(t, 0u, 0x4420u);          /* the four codes as PRMT selector nibbles */
  const uint32_t diff = prmt(SK_POOL_FWD, 0u, sel) ^ x; /* zero byte <=> the byte is exactly A, C, G or T */
  const uint32_t nz = (((diff & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | diff) & 0x80808080u; /* bit 7 of every non-zero byte */
  const uint32_t inv = nz >> 7;                       /* 0/1 per byte: not ACGT -> N (commonFunc.hpp:103-105) */
  code = (code & ~(inv * 3u)) | (inv << 3);
  const uint32_t n = code | (code >> 4);
  return prmt(n, 0u, 0x4420u);
}
__global__ void __launch_bounds__(256) k_pack_bases(const uint4 *__restrict__ in, uint2 *__restrict__ out, uint64_t n16)
{
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
    const uint4 v = in[i];
    uint2 o;
    o.x = pack4(v.x) | (pack4(v.y) << 16);
    o.y = pack4(v.z) | (pack4(v.w) << 16);
    out[i] = o;
  }
}

/* ---------------------------------------------------------------------------------------------------------------
 * K1
 * ------------------------------------------------------------------------------------------------------------- */
struct sk_ctrl {
  int distinct;
  int overflow;
  int above;       /* some valid canonical hash was > T */
  int has_max;     /* the hash value 0xFFFF...F (the table's empty marker) occurred */
  int max_first, max_last, max_votes;
  int _pad;
};

struct sk_smem_layout {
  uint32_t stage_bytes;  /* per staging buffer */
  uint32_t off_bar, off_keys, off_first, off_last, off_votes, off_order, off_bcnt, off_bstart, off_bfill,
      off_ctrl, off_list_h, off_list_p, total;
};

/* CAP = entries of the per-thread candidate list */
__host__ __device__ inline sk_smem_layout sk_layout(int seg_length, int C, int CAP)
{
  sk_smem_layout L;
  /* nibbles of one segment + 16 (alignment of the bulk copy) + 64 (the last threads read a few words past the end) */
  L.stage_bytes = (uint32_t)((((seg_length + 1) / 2 + 15) & ~15) + 16 + 64);
  uint32_t o = 2 * L.stage_bytes;
  L.off_bar = o; o += 16;
  L.off_keys = o; o += 8u * C;
  L.off_first = o; o += 4u * C;
  L.off_last = o; o += 4u * C;
  L.off_votes = o; o += 4u * C;
  L.off_ctrl = o; o += (uint32_t)sizeof(sk_ctrl);
  o = (o + 15) & ~15u;
  /* the per-thread candidate lists are dead once the table is built; the ordering scratch (order[] + bucket counters)
   * lives in the same bytes */
  const uint32_t lists = (16u + 4u) * SK_THREADS * (uint32_t)CAP;
  const uint32_t ordering = ((2u * C + 15) & ~15u) + 3u * 4u * SK_BUCKETS;
  L.off_list_h = o;                                     /* uint4 {hf, hb} [CAP][SK_THREADS] */
  L.off_list_p = o + 16u * SK_THREADS * (uint32_t)CAP;  /* u32 position   [CAP][SK_THREADS] */
  L.off_order = o;
  L.off_bcnt = o + ((2u * C + 15) & ~15u);
  L.off_bstart = L.off_bcnt + 4u * SK_BUCKETS;
  L.off_bfill = L.off_bstart + 4u * SK_BUCKETS;
  o += lists > ordering ? lists : ordering;
  L.total = (o + 15) & ~15u;
  return L;
}

/* insert one occurrence of canonical hash h at position pos with strand vote sv (+1/-1) */
__device__ __forceinline__ void sk_insert(unsigned long long *keys, int *first, int *last, int *votes,
                                          uint32_t mask, int limit, sk_ctrl *ctrl, uint64_t h, int pos, int sv)
{
  if (h == SK_EMPTY) { /* cannot be a table key; keep it in a dedicated entry (it sorts last) */
    ctrl->has_max = 1;
    atomicMin(&ctrl->max_first, pos);
    atomicMax(&ctrl->max_last, pos);
    atomicAdd(&ctrl->max_votes, sv);
    return;
  }
  uint32_t slot = ((uint32_t)h ^ (uint32_t)(h >> 32)) & mask;
  for (uint32_t probe = 0; probe <= mask; probe++) {
    if (*(volatile int *)&ctrl->overflow) return;
    unsigned long long cur = *(volatile unsigned long long *)&keys[slot];
    if (cur == SK_EMPTY) {
      cur = atomicCAS(&keys[slot], (unsigned long long)SK_EMPTY, (unsigned long long)h);
      if (cur == SK_EMPTY) {
        int d = atomicAdd(&ctrl->distinct, 1) + 1;
        if (d > limit) ctrl->overflow = 1;
        cur = h;
      }
    }
    if (cur == h) {
      atomicMin(&first[slot], pos);
      atomicMax(&last[slot], pos);
      atomicAdd(&votes[slot], sv);
      return;
    }
    slot = (slot + 1) & mask;
  }
  ctrl->overflow = 1;
}

/* one raw candidate (both hashes of a position) -> the table, if it is a valid k-mer with canonical hash <= T */
__device__ __forceinline__ void sk_take(unsigned long long *keys, int *first, int *last, int *votes, uint32_t mask,
                                        int limit, sk_ctrl *ctrl, uint64_t hf, uint64_t hb, int pos, uint64_t T, bool &above)
{
  if (hf == hb) return; /* commonFunc.hpp:234 */
  const bool fwd = hf < hb;
  const uint64_t h = fwd ? hf : hb; /* :237 */
  if (h > T) { above = true; return; }
  sk_insert(keys, first, last, votes, mask, limit, ctrl, h, pos, fwd ? 1 : -1); /* :240 */
}

/* Geometry of the k-mer windows in 32-bit words (see the loop below) */
template <int K>
struct sk_geom {
  static constexpr int NH = (K + 3) / 4;        /* 32-bit words holding K bytes                          */
  static constexpr int TB = K - 4 * (NH - 1);   /* bytes used in the last of them (1..4)                 */
  static constexpr int NWIN = (K + 6) / 4;      /* words spanning the 4 k-mers of one step (K + 3 bytes) */
  static constexpr int ROFF = 4 * NWIN - K;     /* byte offset of the reverse-complement k-mer of d = 0  */
};

/* words [OFF, OFF + K) of the byte string held little-endian in A[0..NWIN): out[j] = bytes OFF+4j.. ; the unused
 * bytes of the last word are zero (PRMT selector 8 = sign of byte 0 replicated; every byte here is ASCII or 0) */
template <int K, int OFF>
__device__ __forceinline__ void sk_extract(const uint32_t (&A)[sk_geom<K>::NWIN], uint32_t (&out)[sk_geom<K>::NH])
{
  constexpr int NH = sk_geom<K>::NH, TB = sk_geom<K>::TB, NWIN = sk_geom<K>::NWIN;
#pragma unroll
  for (int j = 0; j < NH; j++) {
    const int b = OFF + 4 * j, wi = b >> 2, bo = b & 3;
    const int nb = (j == NH - 1) ? TB : 4;
    if (bo == 0 && nb == 4) {
      out[j] = A[wi];
    } else {
      uint32_t sel = 0;
#pragma unroll
      for (int t = 0; t < 4; t++) sel |= (uint32_t)(t < nb ? bo + t : 8) << (4 * t);
      const int w2 = (bo + nb > 4 && wi + 1 < NWIN) ? wi + 1 : wi;
      out[j] = prmt(A[wi], A[w2], sel);
    }
  }
}

template <int K>
__device__ __forceinline__ uint64_t sk_hash_words(const uint32_t (&h)[sk_geom<K>::NH])
{
  constexpr int NW = mm_kmer_words<K>::NW;
  uint64_t w[NW];
#pragma unroll
  for (int i = 0; i < NW; i++) w[i] = mm_pack64(h[2 * i], (2 * i + 1 < sk_geom<K>::NH) ? h[2 * i + 1] : 0u);
  return mm_murmur3_k<K>(w);
}

/* per-segment state handed to the hashing loop */
struct sk_run {
  const uint32_t *nib;  /* staged nibbles as aligned 32-bit words (8 bases each) */
  uint32_t b0;          /* base index (within the stage) of this thread's first position */
  int p0, p1;           /* this thread's positions [p0, p1) */
  uint32_t T_hi;
  uint4 *list_h;        /* this thread's column of the candidate list */
  uint32_t *list_p;
  int cap;
};

/* The hashing loop of one thread. CHECK_N: the stretch contains an N -> per-position validity (run of non-N bases >= K).
 * Returns the number of candidates stored (<= cap); candidates beyond cap go straight into the table. */
/* what the hashing loop does with a candidate that no longer fits in the thread's list */
struct sk_spill_table { /* general kernel: straight into the table */
  unsigned long long *keys; int *first, *last, *votes; uint32_t mask; int limit; sk_ctrl *ctrl; uint64_t T; bool *above;
  __device__ __forceinline__ void operator()(uint64_t hf, uint64_t hb, int pos) const
  {
    sk_take(keys, first, last, votes, mask, limit, ctrl, hf, hb, pos, T, *above);
  }
};
struct sk_spill_list { /* fast kernel: a small CTA-wide list; when that is full too the segment goes to the general kernel */
  uint4 *h; uint32_t *p; int *n; int cap;
  __device__ __forceinline__ void operator()(uint64_t hf, uint64_t hb, int pos) const
  {
    const int at = atomicAdd(n, 1);
    if (at < cap) {
      uint32_t fl, fh, bl, bh;
      mm_unpack64(hf, fl, fh);
      mm_unpack64(hb, bl, bh);
      h[at] = make_uint4(fl, fh, bl, bh);
      p[at] = (uint32_t)pos;
    }
  }
};

template <int K, bool CHECK_N, bool TRACK_ABOVE, typename Spill>
__device__ __forceinline__ int sk_hash_run(const sk_run &r, uint32_t &amax, const Spill &spill)
{
  constexpr int NH = sk_geom<K>::NH, NWIN = sk_geom<K>::NWIN, ROFF = sk_geom<K>::ROFF;
  /* F[m] = ASCII of bases 4m..4m+3 after the current step base; C[t] = complement of F-word (NWIN-1-t), byte-reversed,
   * so that C[0] || C[1] || ... is the reverse complement of the NWIN*4 bases read backwards */
  uint32_t F[NWIN], C[NWIN];
  const uint32_t sh = (r.b0 & 7u) * 4u;
  uint32_t wq = r.b0 >> 3;
  uint32_t lo = r.nib[wq], hi = r.nib[wq + 1];
  uint32_t sel = __funnelshift_r(lo, hi, sh); /* the next 8 nibbles, base 0 in bits 0-3 */
  int have = 8;                               /* unused nibbles left in sel */
  auto next_word = [&](uint32_t &f, uint32_t &c) {
    if (have == 0) {
      wq++;
      lo = hi; hi = r.nib[wq + 1];
      sel = __funnelshift_r(lo, hi, sh);
      have = 8;
    }
    f = prmt(SK_POOL_FWD, 0u, sel);                      /* N nibbles (bit 3) give a zero byte */
    c = prmt(prmt(SK_POOL_COMP, 0u, sel), 0u, 0x0123u);  /* complement, bytes reversed */
    sel >>= 16;
    have -= 4;
  };
#pragma unroll
  for (int m = 0; m < NWIN; m++) next_word(F[m], C[NWIN - 1 - m]);

  int run = 0; /* CHECK_N: consecutive non-N bases ending at base (position + K - 2) */
  if (CHECK_N) {
#pragma unroll
    for (int j = 0; j < K - 1; j++) {
      const uint32_t byte = (F[j >> 2] >> (8 * (j & 3))) & 0xFFu;
      run = byte ? run + 1 : 0;
    }
  }
  int cnt = 0;
  uint32_t lofs = 0; /* cnt * SK_THREADS */

  /* the candidate test of one position: its two hashes were computed before (all four positions of a step are hashed
   * first, in straight-line code, so that the eight independent Murmur3 chains overlap; the tests follow) */
  auto consider = [&](uint64_t hf, uint64_t hb, int pos, uint32_t last_byte) {
    bool ok = pos < r.p1;
    if (CHECK_N) {
      run = last_byte ? run + 1 : 0;
      ok = ok && run >= K;
    }
    const uint32_t mh = min((uint32_t)(hf >> 32), (uint32_t)(hb >> 32));
    if (TRACK_ABOVE && ok) amax = max(amax, mh);
    if (ok && mh <= r.T_hi) {
      if (cnt < r.cap) {
        uint32_t fl, fh, bl, bh;
        mm_unpack64(hf, fl, fh);
        mm_unpack64(hb, bl, bh);
        r.list_h[lofs] = make_uint4(fl, fh, bl, bh);
        r.list_p[lofs] = (uint32_t)pos;
        lofs += SK_THREADS;
        cnt++;
      } else {
        spill(hf, hb, pos);
      }
    }
  };

#pragma unroll 1
  for (int p = r.p0; p < r.p1; p += 4) {
    uint32_t fw[NH], rw[NH];
    uint64_t hf0, hb0, hf1, hb1, hf2, hb2, hf3, hb3;
    /* last byte of the forward k-mer of offset d = byte K-1+d of F */
#define SK_LASTB(d) ((F[(K - 1 + (d)) >> 2] >> (8 * ((K - 1 + (d)) & 3))) & 0xFFu)
    const uint32_t lb0 = CHECK_N ? SK_LASTB(0) : 1u, lb1 = CHECK_N ? SK_LASTB(1) : 1u, lb2 = CHECK_N ? SK_LASTB(2) : 1u,
                   lb3 = CHECK_N ? SK_LASTB(3) : 1u;
#undef SK_LASTB
    sk_extract<K, 0>(F, fw); hf0 = sk_hash_words<K>(fw); sk_extract<K, ROFF - 0>(C, rw); hb0 = sk_hash_words<K>(rw);
    sk_extract<K, 1>(F, fw); hf1 = sk_hash_words<K>(fw); sk_extract<K, ROFF - 1>(C, rw); hb1 = sk_hash_words<K>(rw);
    sk_extract<K, 2>(F, fw); hf2 = sk_hash_words<K>(fw); sk_extract<K, ROFF - 2>(C, rw); hb2 = sk_hash_words<K>(rw);
    sk_extract<K, 3>(F, fw); hf3 = sk_hash_words<K>(fw); sk_extract<K, ROFF - 3>(C, rw); hb3 = sk_hash_words<K>(rw);
    consider(hf0, hb0, p + 0, lb0);
    consider(hf1, hb1, p + 1, lb1);
    consider(hf2, hb2, p + 2, lb2);
    consider(hf3, hb3, p + 3, lb3);
    /* slide by one word */
#pragma unroll
    for (int m = 0; m < NWIN - 1; m++) F[m] = F[m + 1];
#pragma unroll
    for (int t = NWIN - 1; t > 0; t--) C[t] = C[t - 1];
    next_word(F[NWIN - 1], C[0]);
  }
  return cnt;
}

/* initial threshold for a segment of n k-mer positions: expect c*S distinct survivors, c = 1.1 + 6/sqrt(S). The canonical hash
 * is the MIN of two uniform hashes, so P(canonical <= t) = 1 - (1-t)^2: solve that for the wanted fraction f = c*S/n.
 * Double-precision sqrt and divide: a few hundred instructions, so the kernels evaluate it once for the usual length
 * (seg_length) and again only for the segments that differ. */
__device__ __forceinline__ uint64_t sk_threshold(int S, int n)
{
  uint64_t T = SK_EMPTY;
  if (n > 0) {
    const double c = 1.1 + 6.0 / sqrt((double)S);
    const double f = c * (double)S / (double)n;
    if (f < 1.0) T = (uint64_t)((1.0 - sqrt(1.0 - f)) * 18446744073709551616.0);
  }
  return T;
}

/* Does any base this thread's k-mers cover carry the N flag (nibble bit 3)? Exactly the bases [b0, b0 + positions + K - 1):
 * the nibbles before and after them in the first / last word are masked off. (Scanning whole words, or a few bases too
 * many, is not harmless: in a packed batch every read is padded with N nibbles up to a multiple of 32 bases, so the last
 * thread of a read's last fragment would take the N-tracking variant of the hashing loop -- and its warp both variants.) */
__device__ __forceinline__ bool sk_any_n(const uint32_t *nib, uint32_t b0, uint32_t n_bases)
{
  if (n_bases == 0) return false;
  const uint32_t e = b0 + n_bases - 1u; /* last base */
  const uint32_t w0 = b0 >> 3, w1 = e >> 3;
  const uint32_t m0 = 0xFFFFFFFFu << ((b0 & 7u) * 4u), m1 = 0xFFFFFFFFu >> ((7u - (e & 7u)) * 4u);
  if (w0 == w1) return (nib[w0] & m0 & m1 & 0x88888888u) != 0;
  uint32_t acc = (nib[w0] & m0) | (nib[w1] & m1);
  for (uint32_t w = w0 + 1; w < w1; w++) acc |= nib[w];
  return (acc & 0x88888888u) != 0;
}

/* sk_val[r] = the lookup-table value of hs[r] for r < count (K2's probe, done here so that its DRAM latency overlaps the
 * other CTAs' hashing). The first slot of every hash is loaded before any is resolved: one round trip per segment for
 * count <= SK_PROBE_BATCH * SK_THREADS. Linear-probe continuations are followed one by one (rare). */
constexpr int SK_PROBE_BATCH = 2;
__device__ __forceinline__ void sk_probe(const mm_tab_slot *__restrict__ tab, int tab_log2, const uint64_t *hs,
                                         uint64_t *__restrict__ sk_val, int count, int tid)
{
  for (int r0 = 0; r0 < count; r0 += SK_PROBE_BATCH * SK_THREADS) {
    uint64_t h[SK_PROBE_BATCH], key[SK_PROBE_BATCH], val[SK_PROBE_BATCH];
    uint32_t slot[SK_PROBE_BATCH];
#pragma unroll
    for (int u = 0; u < SK_PROBE_BATCH; u++) {
      const int r = r0 + u * SK_THREADS + tid;
      if (r < count) {
        h[u] = hs[r];
        slot[u] = mm_tab_slot_of(h[u], tab_log2);
        key[u] = tab[slot[u]].key;
        val[u] = tab[slot[u]].val;
      }
    }
#pragma unroll
    for (int u = 0; u < SK_PROBE_BATCH; u++) {
      const int r = r0 + u * SK_THREADS + tid;
      if (r < count) sk_val[r] = mm_tab_resolve(tab, tab_log2, h[u], slot[u], key[u], val[u]);
    }
  }
}

/* The general kernel: handles every input (any number of repeated k-mers, fewer than s distinct k-mers, thresholds that
 * have to be re-estimated). work_list == nullptr: all n_segs segments; else the segments listed there, *work_count of them
 * (the fast kernel's rejects; the count is read on the device, no host round trip). */
template <int K>
__global__ void __launch_bounds__(SK_THREADS)
k_sketch_table(const uint8_t *__restrict__ packed, const mm_segment *__restrict__ segs, uint32_t n_segs_all,
               const uint32_t *__restrict__ work_list, const uint32_t *__restrict__ work_count, int S,
               int seg_length, int C, int CAP, uint64_t *__restrict__ sk_hash, int2 *__restrict__ sk_pos,
               int8_t *__restrict__ sk_strand, int32_t *__restrict__ sk_votes, mm_segment_result *__restrict__ seg_res,
               const mm_tab_slot *__restrict__ tab, int tab_log2, uint64_t *__restrict__ sk_val)
{
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t n_segs = work_list ? *work_count : n_segs_all;
  const sk_smem_layout L = sk_layout(seg_length, C, CAP);
  uint64_t *bars = (uint64_t *)(smem + L.off_bar);
  unsigned long long *keys = (unsigned long long *)(smem + L.off_keys);
  int *first = (int *)(smem + L.off_first);
  int *last = (int *)(smem + L.off_last);
  int *votes = (int *)(smem + L.off_votes);
  uint16_t *order = (uint16_t *)(smem + L.off_order);
  uint32_t *bcnt = (uint32_t *)(smem + L.off_bcnt);
  uint32_t *bstart = (uint32_t *)(smem + L.off_bstart);
  uint32_t *bfill = (uint32_t *)(smem + L.off_bfill);
  sk_ctrl *ctrl = (sk_ctrl *)(smem + L.off_ctrl);
  const int tid = threadIdx.x;
  uint4 *list_h = (uint4 *)(smem + L.off_list_h) + tid;
  uint32_t *list_p = (uint32_t *)(smem + L.off_list_p) + tid;

  const uint32_t mask = (uint32_t)C - 1;
  const int limit = C / 2;

  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_proxy_async();
  }
  __syncthreads();

  /* nibble bytes of segment seg: [off/2, (off+len+1)/2), copied from the 16-byte floor */
  auto issue = [&](uint32_t seg, int stage) {
    const uint64_t off = segs[seg].offset;
    const int len = segs[seg].length;
    const uint64_t g0 = (off >> 1) & ~15ULL;
    const uint32_t bytes = (uint32_t)(((((off + (uint64_t)len + 1ULL) >> 1) + 15ULL) & ~15ULL) - g0);
    mbar_expect_tx(&bars[stage], bytes);
    bulk_g2s(smem + (size_t)stage * L.stage_bytes, packed + g0, bytes, &bars[stage]);
  };

  const int n_usual = seg_length - K + 1;
  const uint64_t T_usual = sk_threshold(S, n_usual);
  uint32_t it = 0;
  if (tid == 0 && blockIdx.x < n_segs) issue(work_list ? work_list[blockIdx.x] : blockIdx.x, 0);

  for (uint32_t wi = blockIdx.x; wi < n_segs; wi += gridDim.x, it++) {
    const uint32_t seg = work_list ? work_list[wi] : wi;
    const int stage = it & 1;
    const uint32_t next = wi + gridDim.x;
    if (tid == 0 && next < n_segs) {
      fence_proxy_async(); /* generic-proxy reads of that buffer (previous iteration) before the async write */
      issue(work_list ? work_list[next] : next, stage ^ 1);
    }
    const uint64_t off = segs[seg].offset;
    const int len = segs[seg].length;
    const uint32_t skew = (uint32_t)(off - (((off >> 1) & ~15ULL) << 1)); /* bases between the copy's start and the segment */

    const int n = len - K + 1; /* number of k-mer positions (commonFunc.hpp:217) */
    /* positions in steps of four; every thread gets a whole number of steps */
    const int P = n > 0 ? 4 * ((((n + 3) >> 2) + SK_THREADS - 1) / SK_THREADS) : 0;
    sk_run r;
    r.nib = (const uint32_t *)(smem + (size_t)stage * L.stage_bytes);
    r.p0 = tid * P;
    r.p1 = min(n, r.p0 + P);
    r.b0 = skew + (uint32_t)r.p0;
    r.list_h = list_h; r.list_p = list_p; r.cap = CAP;
    const bool has_work = r.p0 < r.p1;

    uint64_t T = n == n_usual ? T_usual : sk_threshold(S, n);
    uint64_t lo = 0, hi = 0;
    bool have_lo = false, have_hi = false;
    bool waited = false;
    bool any_n = false;

    while (true) {
      { /* reset the table: 16-byte stores */
        uint4 *k4 = (uint4 *)keys;
        for (int i = tid; i < C / 2; i += SK_THREADS) k4[i] = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
        int4 *f4 = (int4 *)first, *l4 = (int4 *)last, *v4 = (int4 *)votes;
        for (int i = tid; i < C / 4; i += SK_THREADS) {
          f4[i] = make_int4(0x7fffffff, 0x7fffffff, 0x7fffffff, 0x7fffffff);
          l4[i] = make_int4(-1, -1, -1, -1);
          v4[i] = make_int4(0, 0, 0, 0);
        }
      }
      if (tid == 0) {
        ctrl->distinct = 0; ctrl->overflow = 0; ctrl->above = 0; ctrl->has_max = 0;
        ctrl->max_first = 0x7fffffff; ctrl->max_last = -1; ctrl->max_votes = 0;
      }
      if (!waited) {
        mbar_wait(&bars[stage], (it >> 1) & 1);
        waited = true;
        if (has_work) any_n = sk_any_n(r.nib, r.b0, (uint32_t)(r.p1 - r.p0) + (uint32_t)K - 1u);
      }
      __syncthreads();

      r.T_hi = (uint32_t)(T >> 32);
      bool above = false;
      uint32_t amax = 0;
      int cnt = 0;
      if (has_work) {
        const sk_spill_table spill{keys, first, last, votes, mask, limit, ctrl, T, &above};
        if (any_n) cnt = sk_hash_run<K, true, true>(r, amax, spill);
        else cnt = sk_hash_run<K, false, true>(r, amax, spill);
      }
      if (amax > r.T_hi) above = true; /* a valid position whose smaller hash is certainly > T */
      /* every thread inserts its own candidates */
      for (int q = 0; q < cnt; q++) {
        const uint4 e = list_h[(size_t)q * SK_THREADS];
        const int pos = (int)list_p[(size_t)q * SK_THREADS];
        sk_take(keys, first, last, votes, mask, limit, ctrl, mm_pack64(e.x, e.y), mm_pack64(e.z, e.w), pos, T, above);
      }
      if (above) ctrl->above = 1;
      __syncthreads();
      const int d = ctrl->distinct + ctrl->has_max;
      const int ovf = ctrl->overflow;
      const int abv = ctrl->above;
      if (ovf) { /* too many survivors: lower T */
        hi = T; have_hi = true;
        T = have_lo ? lo + (hi - lo) / 2 : T / 2;
      } else if (d < S && abv) { /* too few: raise T */
        lo = T; have_lo = true;
        if (have_hi) T = lo + (hi - lo) / 2;
        else T = (T > (SK_EMPTY >> 2)) ? SK_EMPTY : (T << 2) | 3ULL;
      } else {
        break;
      }
      __syncthreads();
    }

    /* ---- order the survivors: counting sort on the leading bits, rank inside the bucket ---- */
    const int dt = ctrl->distinct; /* entries in the table (excludes the has_max entry) */
    for (int i = tid; i < SK_BUCKETS; i += SK_THREADS) { bcnt[i] = 0; bfill[i] = 0; } /* aliases the (consumed) lists */
    __syncthreads();
    const int sh = max(0, (64 - __clzll((long long)T)) - 8);
    for (int i = tid; i < C; i += SK_THREADS) {
      const uint64_t k = keys[i];
      if (k != SK_EMPTY) atomicAdd(&bcnt[(uint32_t)(k >> sh)], 1u);
    }
    __syncthreads();
    if (tid < 32) { /* exclusive prefix over 256 buckets by one warp */
      uint32_t loc[SK_BUCKETS / 32];
      uint32_t sum = 0;
#pragma unroll
      for (int j = 0; j < SK_BUCKETS / 32; j++) { loc[j] = sum; sum += bcnt[tid * (SK_BUCKETS / 32) + j]; }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (tid >= o) incl += v;
      }
      const uint32_t excl = incl - sum;
#pragma unroll
      for (int j = 0; j < SK_BUCKETS / 32; j++) bstart[tid * (SK_BUCKETS / 32) + j] = excl + loc[j];
    }
    __syncthreads();
    for (int i = tid; i < C; i += SK_THREADS) {
      const uint64_t k = keys[i];
      if (k != SK_EMPTY) {
        const uint32_t b = (uint32_t)(k >> sh);
        const uint32_t p = bstart[b] + atomicAdd(&bfill[b], 1u);
        order[p] = (uint16_t)i;
      }
    }
    __syncthreads();
    const size_t obase = (size_t)seg * (size_t)S;
    for (int p = tid; p < dt; p += SK_THREADS) {
      const uint32_t slot = order[p];
      const uint64_t k = keys[slot];
      const uint32_t b = (uint32_t)(k >> sh);
      const uint32_t bs = bstart[b], be = bs + bcnt[b];
      uint32_t rank = bs;
      for (uint32_t q = bs; q < be; q++) rank += (keys[order[q]] < k) ? 1u : 0u;
      if ((int)rank < S) {
        sk_hash[obase + rank] = k;
        sk_pos[obase + rank] = make_int2(first[slot], last[slot]);
        const int v = votes[slot];
        sk_strand[obase + rank] = (int8_t)(v > 0 ? 1 : (v == 0 ? 0 : -1)); /* commonFunc.hpp:282 */
        if (sk_votes) sk_votes[obase + rank] = v;
      }
    }
    if (tid == 0) {
      int count = dt;
      if (ctrl->has_max) {
        if (dt < S) {
          sk_hash[obase + dt] = SK_EMPTY;
          sk_pos[obase + dt] = make_int2(ctrl->max_first, ctrl->max_last);
          const int v = ctrl->max_votes;
          sk_strand[obase + dt] = (int8_t)(v > 0 ? 1 : (v == 0 ? 0 : -1));
          if (sk_votes) sk_votes[obase + dt] = v;
        }
        count = dt + 1;
      }
      if (count > S) count = S;
      mm_segment_result res;
      res.sketch_max_hash = 0; /* filled by the L1 kernel from sk_hash[count-1] */
      res.sketch_raw_count = count;
      res.sketch_size = count;
      res.n_points = 0; res.minimum_hits = 0; res.best_intersection = 0;
      res.first_candidate = 0; res.n_candidates = 0; res._pad = 0;
      seg_res[seg] = res;
    }
    if (sk_val) { /* the hashes just written, read back by the whole CTA */
      const int count = min(dt + ctrl->has_max, S);
      __syncthreads();
      sk_probe(tab, tab_log2, sk_hash + obase, sk_val + obase, count, tid);
    }
    __syncthreads(); /* all reads of the staging buffer and of the table are done */
  }
}


/* ---- the fast kernel ------------------------------------------------------------------------------------------
 * One pass per segment, no table, no atomics on the hot path, no threshold loop:
 *   hashing loop (as above) -> per-thread candidate lists;
 *   compaction: every thread filters its own candidates exactly (valid k-mer, canonical hash <= T) and writes them to a
 *     dense array at an offset from a CTA-wide prefix sum;
 *   256-bucket counting sort on the leading bits of the hash (bucket sizes ~1.3);
 *   every thread takes whole buckets: it sorts the bucket by hash (insertion sort of its order[] entries) and counts the
 *     distinct hashes;
 *   a prefix sum over the buckets' distinct counts gives each bucket's first rank; the bucket's owner walks the sorted
 *     bucket again, merges each run of equal hashes into first position / last position / vote sum, writes ranks < s and
 *     looks each written hash up in the index's lookup table (K2's probe).
 * Anything unusual -- more candidates than the dense array holds, a bucket with more than SKF_BUCKET_MAX entries (heavily
 * repeated k-mers), fewer than s distinct hashes below T -- sends the segment to the general kernel through a device
 * work list. On random or genomic sequence that is a fraction of a per cent of the segments.
 */
constexpr int SKF_SPILL = 64;       /* CTA-wide list for candidates that did not fit a thread's own list */
constexpr int SKF_BUCKET_MAX = 24;

struct skf_layout {
  uint32_t stage_bytes, off_bar, off_ctrl, off_list_h, off_spill_h, off_spill_p, off_cand_h, off_cand_m, off_order,
      off_list_p, off_bcnt, total;
};
struct skf_ctrl {
  int n_spill, n_cand, reject, warp_tot[SK_THREADS / 32];
};
__host__ __device__ inline skf_layout skf_make_layout(int seg_length, int NC, int CAP)
{
  skf_layout L;
  L.stage_bytes = (uint32_t)((((seg_length + 1) / 2 + 15) & ~15) + 16 + 64);
  uint32_t o = 2 * L.stage_bytes;
  L.off_bar = o; o += 16;
  L.off_ctrl = o; o += 2 * 32; /* two copies, used alternately (see the kernel) */
  L.off_spill_h = o; o += 16u * SKF_SPILL;
  L.off_spill_p = o; o += 4u * SKF_SPILL;
  L.off_cand_h = o; o += 8u * NC;   /* canonical hash */
  L.off_cand_m = o; o += 4u * NC;   /* position << 1 | (forward hash was the smaller one) */
  /* the per-thread lists are dead after the compaction: order[] and five bucket counter arrays (bcnt, bstart, bfill, dcnt,
   * dstart: SK_BUCKETS u32 each, addressed by constant offsets from bcnt) live in the same bytes */
  const uint32_t lists = (16u + 4u) * SK_THREADS * (uint32_t)CAP;
  const uint32_t sorting = ((2u * NC + 15) & ~15u) + 5u * 4u * SK_BUCKETS;
  L.off_list_h = o;
  L.off_list_p = o + 16u * SK_THREADS * (uint32_t)CAP;
  L.off_order = o;
  L.off_bcnt = o + ((2u * NC + 15) & ~15u);
  o += lists > sorting ? lists : sorting;
  L.total = (o + 15) & ~15u;
  return L;
}

/* exclusive prefix over SK_BUCKETS counters by warp 0 */
__device__ __forceinline__ void skf_bucket_prefix(const uint32_t *cnt, uint32_t *start, int tid)
{
  if (tid < 32) {
    uint32_t loc[SK_BUCKETS / 32];
    uint32_t sum = 0;
#pragma unroll
    for (int j = 0; j < SK_BUCKETS / 32; j++) { loc[j] = sum; sum += cnt[tid * (SK_BUCKETS / 32) + j]; }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (tid >= o) incl += v;
    }
    const uint32_t excl = incl - sum;
#pragma unroll
    for (int j = 0; j < SK_BUCKETS / 32; j++) start[tid * (SK_BUCKETS / 32) + j] = excl + loc[j];
  }
}

template <int K>
__global__ void __launch_bounds__(SK_THREADS, MM_SK_MINB)
k_sketch(const uint8_t *__restrict__ packed, const mm_segment *__restrict__ segs, uint32_t n_segs, int S, int seg_length,
         int NC, int CAP, uint64_t *__restrict__ sk_hash, int2 *__restrict__ sk_pos, int8_t *__restrict__ sk_strand,
         mm_segment_result *__restrict__ seg_res, uint32_t *__restrict__ reject_list, uint32_t *__restrict__ reject_count,
         const mm_tab_slot *__restrict__ tab, int tab_log2, uint64_t *__restrict__ sk_val)
{
  extern __shared__ __align__(16) unsigned char smem[];
  const skf_layout L = skf_make_layout(seg_length, NC, CAP);
  uint64_t *bars = (uint64_t *)(smem + L.off_bar);
  skf_ctrl *ctrl2 = (skf_ctrl *)(smem + L.off_ctrl);
  static_assert(sizeof(skf_ctrl) <= 32, "skf_ctrl");
  uint4 *spill_h = (uint4 *)(smem + L.off_spill_h);
  uint32_t *spill_p = (uint32_t *)(smem + L.off_spill_p);
  uint64_t *cand_h = (uint64_t *)(smem + L.off_cand_h);
  uint32_t *cand_m = (uint32_t *)(smem + L.off_cand_m);
  uint16_t *order = (uint16_t *)(smem + L.off_order);
  uint32_t *bcnt = (uint32_t *)(smem + L.off_bcnt);
  uint32_t *bstart = bcnt + SK_BUCKETS, *bfill = bcnt + 2 * SK_BUCKETS, *dcnt = bcnt + 3 * SK_BUCKETS,
           *dstart = bcnt + 4 * SK_BUCKETS;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  uint4 *list_h = (uint4 *)(smem + L.off_list_h) + tid;
  uint32_t *list_p = (uint32_t *)(smem + L.off_list_p) + tid;

  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_proxy_async();
    ctrl2[0].n_spill = 0; ctrl2[0].reject = 0;
    ctrl2[1].n_spill = 0; ctrl2[1].reject = 0;
  }
  __syncthreads();

  auto issue = [&](uint32_t seg, int stage) {
    const uint64_t off = segs[seg].offset;
    const int len = segs[seg].length;
    const uint64_t g0 = (off >> 1) & ~15ULL;
    const uint32_t bytes = (uint32_t)(((((off + (uint64_t)len + 1ULL) >> 1) + 15ULL) & ~15ULL) - g0);
    mbar_expect_tx(&bars[stage], bytes);
    bulk_g2s(smem + (size_t)stage * L.stage_bytes, packed + g0, bytes, &bars[stage]);
  };

  const int n_usual = seg_length - K + 1;
  const uint64_t T_usual = sk_threshold(S, n_usual);
  uint32_t it = 0;
  if (tid == 0 && blockIdx.x < n_segs) issue(blockIdx.x, 0);

  for (uint32_t seg = blockIdx.x; seg < n_segs; seg += gridDim.x, it++) {
    const int stage = it & 1;
    /* the spill counter / reject flag are written during one segment's hashing loop by threads that may be a whole
     * phase ahead of thread 0: two copies used alternately, the idle one is cleared in the middle of the other's turn */
    skf_ctrl *ctrl = ctrl2 + (it & 1), *ctrl_next = ctrl2 + ((it + 1) & 1);
    const uint32_t next = seg + gridDim.x;
    if (tid == 0 && next < n_segs) {
      fence_proxy_async();
      issue(next, stage ^ 1);
    }
    const uint64_t off = segs[seg].offset;
    const int len = segs[seg].length;
    const uint32_t skew = (uint32_t)(off - (((off >> 1) & ~15ULL) << 1));
    const int n = len - K + 1;
    const int P = n > 0 ? 4 * ((((n + 3) >> 2) + SK_THREADS - 1) / SK_THREADS) : 0;
    sk_run r;
    r.nib = (const uint32_t *)(smem + (size_t)stage * L.stage_bytes);
    r.p0 = tid * P;
    r.p1 = min(n, r.p0 + P);
    r.b0 = skew + (uint32_t)r.p0;
    r.list_h = list_h; r.list_p = list_p; r.cap = CAP;
    const bool has_work = r.p0 < r.p1;
    const uint64_t T = n == n_usual ? T_usual : sk_threshold(S, n);
    r.T_hi = (uint32_t)(T >> 32);

    mbar_wait(&bars[stage], (it >> 1) & 1);
    int cnt = 0;
    if (has_work) {
      uint32_t amax = 0;
      const sk_spill_list spill{spill_h, spill_p, &ctrl->n_spill, SKF_SPILL};
      if (sk_any_n(r.nib, r.b0, (uint32_t)(r.p1 - r.p0) + (uint32_t)K - 1u)) cnt = sk_hash_run<K, true, false>(r, amax, spill);
      else cnt = sk_hash_run<K, false, false>(r, amax, spill);
    }

    /* ---- compaction: exact filter, CTA-wide prefix sum, dense (hash, position|strand) array ---- */
    int keep = 0;
    uint32_t keep_mask = 0;
    for (int q = 0; q < cnt; q++) {
      const uint4 e = list_h[(size_t)q * SK_THREADS];
      const uint64_t hf = mm_pack64(e.x, e.y), hb = mm_pack64(e.z, e.w);
      const uint64_t h = hf < hb ? hf : hb;
      if (hf != hb && h <= T) { keep++; keep_mask |= 1u << q; }
    }
    int incl = keep;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) ctrl->warp_tot[wid] = incl;
    __syncthreads();
    if (tid == 0) { ctrl_next->n_spill = 0; ctrl_next->reject = 0; } /* nobody is in the next segment's loop yet, nobody in the last one's */
    int base = incl - keep;
    for (int w = 0; w < wid; w++) base += ctrl->warp_tot[w];
    int total = 0;
#pragma unroll
    for (int w = 0; w < SK_THREADS / 32; w++) total += ctrl->warp_tot[w];
    const int n_spill = min(ctrl->n_spill, SKF_SPILL);
    const bool spill_over = ctrl->n_spill > SKF_SPILL;
    /* the lists are read and the dense array is written in the same pass; the dense array does not alias the lists */
    if (total + n_spill <= NC) {
      int at = base;
      for (int q = 0; q < cnt; q++) {
        if (keep_mask & (1u << q)) {
          const uint4 e = list_h[(size_t)q * SK_THREADS];
          const uint64_t hf = mm_pack64(e.x, e.y), hb = mm_pack64(e.z, e.w);
          const bool fwd = hf < hb;
          cand_h[at] = fwd ? hf : hb;
          cand_m[at] = (list_p[(size_t)q * SK_THREADS] << 1) | (fwd ? 1u : 0u);
          at++;
        }
      }
    }
    __syncthreads(); /* lists consumed: their bytes become order[] / counters */
    bool reject = spill_over || total + n_spill > NC;
    int nc = total;
    if (!reject) {
      /* spilled candidates (rare): thread 0 appends them */
      if (n_spill) {
        if (tid == 0) {
          int at = total;
          for (int q = 0; q < n_spill; q++) {
            const uint4 e = spill_h[q];
            const uint64_t hf = mm_pack64(e.x, e.y), hb = mm_pack64(e.z, e.w);
            const bool fwd = hf < hb;
            const uint64_t h = fwd ? hf : hb;
            if (hf != hb && h <= T) { cand_h[at] = h; cand_m[at] = (spill_p[q] << 1) | (fwd ? 1u : 0u); at++; }
          }
          ctrl->n_cand = at;
        }
      }
      for (int i = tid; i < SK_BUCKETS; i += SK_THREADS) { bcnt[i] = 0; bfill[i] = 0; }
      __syncthreads();
      if (n_spill) nc = ctrl->n_cand;
      const int sh = max(0, (64 - __clzll((long long)T)) - 8);
      for (int i = tid; i < nc; i += SK_THREADS) atomicAdd(&bcnt[(uint32_t)(cand_h[i] >> sh)], 1u);
      __syncthreads();
      skf_bucket_prefix(bcnt, bstart, tid);
      __syncthreads();
      for (int i = tid; i < nc; i += SK_THREADS) {
        const uint32_t b = (uint32_t)(cand_h[i] >> sh);
        order[bstart[b] + atomicAdd(&bfill[b], 1u)] = (uint16_t)i;
      }
      __syncthreads();
      /* one thread per bucket: order it by hash, count its distinct hashes */
      bool big_bucket = false;
      for (int b = tid; b < SK_BUCKETS; b += SK_THREADS) {
        const uint32_t bs = bstart[b], be = bs + bcnt[b];
        uint32_t nd = be - bs;
        if (nd > (uint32_t)SKF_BUCKET_MAX) {
          big_bucket = true;
        } else if (nd > 1) {
          for (uint32_t q = bs + 1; q < be; q++) {
            const uint16_t j = order[q];
            const uint64_t h = cand_h[j];
            uint32_t p = q;
            for (; p > bs && cand_h[order[p - 1]] > h; p--) order[p] = order[p - 1];
            order[p] = j;
          }
          uint64_t prev = cand_h[order[bs]];
          nd = 1;
          for (uint32_t q = bs + 1; q < be; q++) {
            const uint64_t h = cand_h[order[q]];
            nd += h != prev ? 1u : 0u;
            prev = h;
          }
        }
        dcnt[b] = nd;
      }
      if (big_bucket) ctrl->reject = 1;
      __syncthreads();
      skf_bucket_prefix(dcnt, dstart, tid);
      __syncthreads();
      const int distinct = (int)(dstart[SK_BUCKETS - 1] + dcnt[SK_BUCKETS - 1]);
      reject = ctrl->reject != 0 || (distinct < S && T != SK_EMPTY);
      if (!reject) {
        const size_t obase = (size_t)seg * (size_t)S;
        /* each bucket's owner merges the runs of equal hashes (first / last position, vote sum), writes ranks < s and
         * looks each written hash up in the table: the loads of its first two ranks are issued in the walk and resolved
         * after it, any further one at once (a separate probe phase behind one more barrier makes ptxas spill the hashing
         * loop's state) */
        int pr0 = -1, pr1 = -1;
        uint32_t ps0 = 0, ps1 = 0;
        uint64_t ph0 = 0, ph1 = 0, pk0 = 0, pk1 = 0, pv0 = 0, pv1 = 0;
        for (int b = tid; b < SK_BUCKETS; b += SK_THREADS) {
          const uint32_t bs = bstart[b], be = bs + bcnt[b];
          int rank = (int)dstart[b];
          uint32_t q = bs;
          while (q < be && rank < S) {
            const uint64_t h = cand_h[order[q]];
            int first = 0x7fffffff, last = -1, votes = 0;
            for (; q < be; q++) {
              const uint16_t j = order[q];
              if (cand_h[j] != h) break;
              const uint32_t m = cand_m[j];
              const int pj = (int)(m >> 1);
              first = min(first, pj); last = max(last, pj); votes += (m & 1u) ? 1 : -1;
            }
            sk_hash[obase + rank] = h;
            sk_pos[obase + rank] = make_int2(first, last);
            sk_strand[obase + rank] = (int8_t)(votes > 0 ? 1 : (votes == 0 ? 0 : -1)); /* commonFunc.hpp:282 */
            if (sk_val) {
              if (pr0 < 0) {
                pr0 = rank; ph0 = h; ps0 = mm_tab_slot_of(h, tab_log2); pk0 = tab[ps0].key; pv0 = tab[ps0].val;
              } else if (pr1 < 0) {
                pr1 = rank; ph1 = h; ps1 = mm_tab_slot_of(h, tab_log2); pk1 = tab[ps1].key; pv1 = tab[ps1].val;
              } else {
                sk_val[obase + rank] = mm_tab_lookup(tab, tab_log2, h);
              }
            }
            rank++;
          }
        }
        if (pr0 >= 0) sk_val[obase + pr0] = mm_tab_resolve(tab, tab_log2, ph0, ps0, pk0, pv0);
        if (pr1 >= 0) sk_val[obase + pr1] = mm_tab_resolve(tab, tab_log2, ph1, ps1, pk1, pv1);
        const int count = min(distinct, S);
        if (tid == 0) {
          mm_segment_result res;
          res.sketch_max_hash = 0; /* filled by the L1 kernel from sk_hash[count-1] */
          res.sketch_raw_count = count;
          res.sketch_size = count;
          res.n_points = 0; res.minimum_hits = 0; res.best_intersection = 0;
          res.first_candidate = 0; res.n_candidates = 0; res._pad = 0;
          seg_res[seg] = res;
        }
      }
    }
    if (reject && tid == 0) reject_list[atomicAdd(reject_count, 1u)] = seg; /* the general kernel takes it */
    __syncthreads(); /* everything read; the staging buffer, lists and counters may be overwritten */
  }
}

/* table capacity and candidate-list capacity for (seg_length, sketch_size) */
void sk_sizes(int seg_length, int sketch_size, int kmer_size, int *C_out, int *CAP_out)
{
  /* survivors ~ c*S with c = 1.1 + 6/sqrt(S); the table may be half full at most */
  const double c = 1.1 + 6.0 / sqrt((double)sketch_size);
  const double want = 2.0 * (c * sketch_size + 8.0 * sqrt(c * sketch_size) + 16.0);
  int C = 512;
  while (C < want) C <<= 1;
  /* candidates per thread ~ Poisson(mu): mu + 2 sqrt(mu) + 1 entries hold all but a few per cent of the threads'
   * lists; the rest go straight to the table (correct, just slower) */
  const int n = seg_length - kmer_size + 1 > 0 ? seg_length - kmer_size + 1 : 1;
  const int P = 4 * ((((n + 3) >> 2) + SK_THREADS - 1) / SK_THREADS);
  double f = c * (double)sketch_size / (double)n;
  if (f > 1.0) f = 1.0;
  const double mu = f * P;
  int CAP = (int)ceil(mu + 2.0 * sqrt(mu) + 1.0);
  if (CAP < 4) CAP = 4;
  if (CAP > 24) CAP = 24;
  *C_out = C;
  *CAP_out = CAP;
}

/* dense-array capacity of the fast kernel: the expected number of candidates + 6 sigma, at least 256 */
int skf_cand_cap(int seg_length, int sketch_size, int kmer_size)
{
  const double c = 1.1 + 6.0 / sqrt((double)sketch_size);
  const int n = seg_length - kmer_size + 1 > 0 ? seg_length - kmer_size + 1 : 1;
  double want = c * sketch_size;
  if (want > n) want = n;
  int NC = (int)(want + 6.0 * sqrt(want) + 32.0);
  NC = (NC + 63) & ~63;
  return NC < 256 ? 256 : NC;
}

template <int K>
cudaError_t launch_k(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, cudaStream_t st, int sm_count, int C,
                     int CAP, size_t smem, int mode)
{
  /* general kernel: over everything (mode 1, MM_SKETCH_TABLE=1) or over the fast kernel's rejects (mode 0) */
  cudaError_t e = cudaFuncSetAttribute(k_sketch_table<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_sketch_table<K>, SK_THREADS, smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) occ = 1;
  const uint32_t full = (uint32_t)sm_count * (uint32_t)occ;
  if (b.n_segs == 0) return cudaSuccess;
  const int NC = skf_cand_cap(p.seg_length, p.sketch_size, K);
  const skf_layout FL = skf_make_layout(p.seg_length, NC, CAP);
  if (mode == 1 || NC > 65535 || FL.total > 227u * 1024u) {
    const uint32_t grid = full > b.n_segs ? b.n_segs : full;
    k_sketch_table<K><<<grid, SK_THREADS, smem, st>>>(b.packed, b.segs, b.n_segs, nullptr, nullptr, p.sketch_size, p.seg_length, C,
                                                      CAP, b.sk_hash, b.sk_pos, b.sk_strand, b.sk_votes, b.seg_res, ix.tab,
                                                      ix.tab_log2, b.sk_val);
    return cudaGetLastError();
  }
  e = cudaFuncSetAttribute(k_sketch<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FL.total);
  if (e != cudaSuccess) return e;
  int focc = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&focc, k_sketch<K>, SK_THREADS, FL.total);
  if (e != cudaSuccess) return e;
  if (focc < 1) focc = 1;
  uint32_t fgrid = (uint32_t)sm_count * (uint32_t)focc; /* persistent: a whole number of CTAs per SM */
  if (fgrid > b.n_segs) fgrid = b.n_segs;
  k_sketch<K><<<fgrid, SK_THREADS, FL.total, st>>>(b.packed, b.segs, b.n_segs, p.sketch_size, p.seg_length, NC, CAP, b.sk_hash, b.sk_pos,
                                                   b.sk_strand, b.seg_res, b.sk_reject, &b.counters->sketch_rejects, ix.tab,
                                                   ix.tab_log2, b.sk_val);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  /* the rejects: the count is read on the device; a grid of one CTA per SM is enough for a fraction of a per cent */
  uint32_t rgrid = (uint32_t)sm_count;
  if (rgrid > b.n_segs) rgrid = b.n_segs;
  k_sketch_table<K><<<rgrid, SK_THREADS, smem, st>>>(b.packed, b.segs, b.n_segs, b.sk_reject, &b.counters->sketch_rejects,
                                                     p.sketch_size, p.seg_length, C, CAP, b.sk_hash, b.sk_pos, b.sk_strand,
                                                     b.sk_votes, b.seg_res, ix.tab, ix.tab_log2, b.sk_val);
  return cudaGetLastError();
}

/* ---------------------------------------------------------------------------------------------------------------
 * K1 for a fragment longer than seg_length (an unsplit query, --noSplit): it does not fit one CTA's shared memory, so
 * it is cut into pieces of at most seg_length bases, consecutive pieces overlapping by k-1 bases -- every k-mer start
 * position belongs to exactly one piece, and the N test and both hashes of a k-mer read only its own k bases -- the
 * pieces are sketched as ordinary segments by the general kernel above (k_sketch_table, the only one that writes the
 * vote SUMS; the fast kernel stays as it is for the ordinary segments), and merged here.
 *
 * Exactness: let h be one of the s smallest distinct hashes of the whole fragment. In every piece where h occurs, fewer
 * than s distinct hashes of the piece are smaller than h (each is also a hash of the fragment), so h is among the
 * piece's s smallest and the piece reports h with its first and last position and the vote sum of ALL its occurrences
 * in that piece. Over the pieces these cover every occurrence of h: first = min, last = max (plus the piece offset),
 * votes = sum. Every hash the pieces report is a hash of the fragment, so the s smallest distinct hashes of the union
 * are exactly the fragment's s smallest; and where the fragment has fewer than s distinct hashes every piece reports
 * all of its own, so the union is all of them. The union's other (larger) hashes may have partial statistics; they are
 * never written.
 *
 * The merge: one sort of the pieces' slots by hash per fragment (library segmented radix sort, plumbing), then one warp
 * per fragment walks the sorted slots 32 at a time: the first slot of every hash run is a head, a ballot ranks the heads,
 * a head whose rank is < s adds up its run (at most one slot per piece) and writes the fragment's slot `rank`.
 * ------------------------------------------------------------------------------------------------------------- */

/* slot i of the pieces' area: key = its hash, or ~0 where the piece has fewer than s hashes (value i either way, so a
 * padding slot is told apart from a real hash ~0 by its index) */
__global__ void k_long_prep(const mm_segment_result *__restrict__ seg_res, uint64_t *__restrict__ sk_hash, uint32_t piece_base,
                            int S, uint64_t n_entries, uint32_t *__restrict__ vals)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_entries) return;
  const uint64_t slot = (uint64_t)piece_base * (uint64_t)S + i;
  const uint32_t seg = piece_base + (uint32_t)(i / (uint64_t)S);
  if ((int)(i % (uint64_t)S) >= seg_res[seg].sketch_size) sk_hash[slot] = SK_EMPTY;
  vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(128) k_long_merge(const mm_long_frag *__restrict__ frags, uint32_t n_frags,
                                                    const uint64_t *__restrict__ entry_off, const uint64_t *__restrict__ keys,
                                                    const uint32_t *__restrict__ vals, uint32_t piece_base, int S,
                                                    int piece_step, const int32_t *__restrict__ pk_votes,
                                                    uint64_t *__restrict__ sk_hash, int2 *sk_pos, int8_t *__restrict__ sk_strand,
                                                    mm_segment_result *seg_res, const mm_tab_slot *__restrict__ tab, int tab_log2,
                                                    uint64_t *__restrict__ sk_val)
{
  const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (f >= n_frags) return;
  const mm_long_frag fr = frags[f];
  const uint64_t b0 = entry_off[f], b1 = entry_off[f + 1];
  const uint32_t q0 = fr.piece0 - piece_base; /* first piece of this fragment in the pieces' area */
  const size_t obase = (size_t)fr.seg * (size_t)S;
  int rank = 0;
  for (uint64_t base = b0; base < b1 && rank < S; base += 32) {
    const uint64_t i = base + (uint64_t)lane;
    bool head = false;
    uint64_t h = 0;
    if (i < b1) {
      h = keys[i];
      head = i == b0 || keys[i - 1] != h;
    }
    int first = 0x7fffffff, last = -1, votes = 0;
    bool real = false;
    if (head) {
      for (uint64_t t = i; t < b1 && keys[t] == h; t++) {
        const uint32_t v = vals[t];
        const uint32_t q = v / (uint32_t)S, j = v % (uint32_t)S;
        if ((int)j >= seg_res[piece_base + q].sketch_size) continue; /* padding of a piece with fewer than s hashes */
        const uint64_t slot = (uint64_t)piece_base * (uint64_t)S + v;
        const int off = (int)(q - q0) * piece_step;
        const int2 p = sk_pos[slot]; /* a piece's slot: never one the merge writes */
        first = min(first, p.x + off);
        last = max(last, p.y + off);
        votes += pk_votes[slot];
        real = true;
      }
    }
    const uint32_t heads = __ballot_sync(0xffffffffu, real);
    const int r = rank + __popc(heads & ((1u << lane) - 1u));
    if (real && r < S) {
      sk_hash[obase + r] = h;
      sk_pos[obase + r] = make_int2(first, last);
      sk_strand[obase + r] = (int8_t)(votes > 0 ? 1 : (votes == 0 ? 0 : -1)); /* commonFunc.hpp:282 */
      if (sk_val) sk_val[obase + r] = mm_tab_lookup(tab, tab_log2, h);
    }
    rank += __popc(heads);
  }
  if (lane == 0) {
    const int count = min(rank, S);
    mm_segment_result res;
    res.sketch_max_hash = 0;
    res.sketch_raw_count = count;
    res.sketch_size = count;
    res.n_points = 0; res.minimum_hits = 0; res.best_intersection = 0;
    res.first_candidate = 0; res.n_candidates = 0; res._pad = 0;
    seg_res[fr.seg] = res;
  }
}

} // namespace

size_t mm_sketch_long_tmp_bytes(uint64_t n_entries, uint32_t n_frags)
{
  size_t sort_bytes = 0;
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                           (const uint32_t *)nullptr, (uint32_t *)nullptr, (int64_t)n_entries, (int64_t)n_frags,
                                           (const uint64_t *)nullptr, (const uint64_t *)nullptr);
  /* keys out (u64) + values in / out (u32) + the sort's own area */
  return n_entries * 16 + 256 * 3 + sort_bytes;
}

cudaError_t mm_launch_sketch_long_merge(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, const mm_long_frag *frags,
                                        const uint64_t *entry_off, uint32_t n_frags, uint32_t piece_base, uint64_t n_entries,
                                        void *tmp, size_t tmp_bytes, cudaStream_t st)
{
  if (n_frags == 0 || n_entries == 0) return cudaSuccess;
  const int S = p.sketch_size;
  unsigned char *t = (unsigned char *)tmp;
  uint64_t *keys_out = (uint64_t *)t;
  uint32_t *vals_in = (uint32_t *)(t + ((n_entries * 8 + 255) & ~255ULL));
  uint32_t *vals_out = (uint32_t *)((unsigned char *)vals_in + ((n_entries * 4 + 255) & ~255ULL));
  unsigned char *sort_tmp = (unsigned char *)vals_out + ((n_entries * 4 + 255) & ~255ULL);
  size_t sort_bytes = tmp_bytes - (size_t)(sort_tmp - t);
  uint64_t *keys_in = b.sk_hash + (uint64_t)piece_base * (uint64_t)S;
  k_long_prep<<<(uint32_t)((n_entries + 255) / 256), 256, 0, st>>>(b.seg_res, b.sk_hash, piece_base, S, n_entries, vals_in);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  e = cub::DeviceSegmentedRadixSort::SortPairs(sort_tmp, sort_bytes, keys_in, keys_out, vals_in, vals_out, (int64_t)n_entries,
                                               (int64_t)n_frags, entry_off, entry_off + 1, 0, 64, st);
  if (e != cudaSuccess) return e;
  k_long_merge<<<(n_frags + 3) / 4, 128, 0, st>>>(frags, n_frags, entry_off, keys_out, vals_out, piece_base, S,
                                                  p.seg_length - p.kmer_size + 1, b.sk_votes, b.sk_hash, b.sk_pos, b.sk_strand,
                                                  b.seg_res, ix.tab, ix.tab_log2, b.sk_val);
  return cudaGetLastError();
}

#define MM_FOR_EACH_K(X) \
  X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16) X(17) X(18) X(19) X(20) X(21) X(22) X(23) X(24) X(25) X(26) X(27) \
  X(28) X(29) X(30) X(31) X(32)

int mm_sketch_kmer_supported(int k)
{
  switch (k) {
#define X(KK) case KK:
    MM_FOR_EACH_K(X)
#undef X
    return 1;
    default: return 0;
  }
}

size_t mm_sketch_smem_bytes(int seg_length, int sketch_size, int kmer_size, int *table_cap, int *list_cap)
{
  int C = 0, CAP = 0;
  sk_sizes(seg_length, sketch_size, kmer_size, &C, &CAP);
  if (C > 32768) return 0; /* order[] holds 16-bit slots */
  sk_smem_layout L = sk_layout(seg_length, C, CAP);
  while (L.total > 227u * 1024u && CAP > 4) { /* long segments: a shorter list before giving up */
    CAP--;
    L = sk_layout(seg_length, C, CAP);
  }
  if (L.total > 227u * 1024u) return 0;
  if (table_cap) *table_cap = C;
  if (list_cap) *list_cap = CAP;
  return L.total;
}

cudaError_t mm_launch_pack_bases(const uint8_t *ascii, uint8_t *packed, uint64_t n_bases, cudaStream_t st, int sm_count)
{
  const uint64_t n16 = (n_bases + 15) / 16; /* both buffers are padded to a multiple of 16 bases */
  if (n16 == 0) return cudaSuccess;
  uint64_t grid = (n16 + 255) / 256;
  const uint64_t cap = (uint64_t)sm_count * 16;
  if (grid > cap) grid = cap;
  k_pack_bases<<<(uint32_t)grid, 256, 0, st>>>((const uint4 *)ascii, (uint2 *)packed, n16);
  return cudaGetLastError();
}

/* mode 0: fast kernel + general kernel over its rejects (2 launches); mode 1: general kernel over everything (1 launch).
 * b.counters->sketch_rejects must be 0 and b.sk_reject must hold n_segs entries. */
cudaError_t mm_launch_sketch(const mm_params &p, const mm_dev_index &ix, const mm_dev_batch &b, cudaStream_t st, int sm_count,
                             int mode)
{
  int C = 0, CAP = 0;
  const size_t smem = mm_sketch_smem_bytes(p.seg_length, p.sketch_size, p.kmer_size, &C, &CAP);
  if (smem == 0) return cudaErrorInvalidValue;
  switch (p.kmer_size) {
#define X(KK) case KK: return launch_k<KK>(p, ix, b, st, sm_count, C, CAP, smem, mode);
    MM_FOR_EACH_K(X)
#undef X
    default: return cudaErrorInvalidValue;
  }
}
