/*
 * mm_inflate.h -- raw DEFLATE (RFC 1951) decoding of one bounded block, and its CRC-32 (RFC 1952).
 *
 * One statement, compiled __host__ __device__ like mm_winmachine.h: the kernel in mm_inflate.cu runs it with the 32
 * lanes of a warp, the host (skch::seqio's CPU inflater, the tests) with one lane. Every lane runs the whole Huffman
 * decode on the same input and the same tables, so control flow is warp-uniform; lanes split only the work that has
 * no order inside it: counting code lengths, filling the lookup tables, match copies, stored copies and the CRC.
 *
 * Bounds: the decoder reads in[0, in_len) and writes out[0, out_len), nothing else, whatever the input. Bits asked for
 * beyond in_len read as zeros and make the block fail (MMI_E_INPUT) before any of them can move the output past its
 * range. A block is accepted only when the stream ends (BFINAL) on the last byte of its input and fills exactly its
 * output range: any malformed stream ends in a status code, never in a fault.
 */
#ifndef MM_INFLATE_H
#define MM_INFLATE_H

#include <stdint.h>

#if defined(__CUDACC__)
#define MMI_HD __host__ __device__ __forceinline__
#else
#define MMI_HD inline
#endif

enum mmi_status {
  MMI_OK = 0,
  MMI_E_INPUT = 1,    /* the stream needs bits past the block's compressed bytes */
  MMI_E_OUTPUT = 2,   /* the stream inflates to more than the block's output range */
  MMI_E_SHORT = 3,    /* ... or to less */
  MMI_E_BTYPE = 4,    /* block type 3 */
  MMI_E_STORED = 5,   /* stored block whose LEN and NLEN do not match */
  MMI_E_CODES = 6,    /* code lengths that do not make a prefix code (or too many symbols, no end-of-block code) */
  MMI_E_SYMBOL = 7,   /* a bit pattern that is no code, or a length / distance symbol that does not exist */
  MMI_E_DIST = 8,     /* a distance back past the start of the block's output */
  MMI_E_TRAILING = 9, /* the stream ends before the last byte of the block's compressed bytes */
  MMI_E_CRC = 10,     /* inflated text whose CRC-32 differs from the member's (checked by the callers) */
};

#if defined(__CUDACC__)
/* internal to libmashmap_b200.so (mm_fastq.cu inflates BGZF members into its window): k_inflate over n blocks whose
 * arrays are all in device memory, as mm_inflate_blocks lays them out, on stream st; status[i] gets block i's mmi_status
 * (the CRC-32 checked). mmi_status_text says what a status means. */
cudaError_t mmi_launch_inflate(const uint8_t *comp, const uint64_t *coff, const uint64_t *ooff, const uint32_t *crc, uint64_t n,
                               uint8_t *out, int32_t *status, cudaStream_t st);
const char *mmi_status_text(int rc);
#endif

#define MMI_FAST 9 /* lookup-table bits: codes up to 9 bits decode in one table read, longer ones canonically */

template <int N>
struct mmi_huff {
  uint16_t count[16]; /* codes of each length */
  uint16_t sym[N];    /* symbols ordered by (length, value): the canonical order */
};

/* one decoder's tables: ~3.1 KB, in shared memory on the device (one per warp) */
struct mmi_tables {
  mmi_huff<288> lit;
  mmi_huff<32> dist;
  mmi_huff<20> clen;
  uint16_t lfast[1 << MMI_FAST], dfast[1 << MMI_FAST]; /* (length << 9) | symbol, 0 = longer than MMI_FAST */
  uint8_t lens[320];                                   /* literal/length then distance code lengths */
  uint8_t clens[20];                                   /* code-length code lengths */
};

MMI_HD void mmi_sync()
{
#if defined(__CUDA_ARCH__)
  __syncwarp();
#endif
}

/* LSB-first bit reader; the consumed bit position is pos * 8 - cnt, where pos also counts the zero bytes read past in_len */
struct mmi_bits {
  const uint8_t *in;
  uint64_t len, pos;
  uint64_t buf;
  int cnt;
  MMI_HD void refill()
  {
    while (cnt <= 56) {
      buf |= (uint64_t)(pos < len ? in[pos] : 0) << cnt;
      pos++;
      cnt += 8;
    }
  }
  MMI_HD uint32_t take(int n) /* n <= cnt */
  {
    const uint32_t v = (uint32_t)(buf & ((1ULL << n) - 1));
    buf >>= n;
    cnt -= n;
    return v;
  }
  MMI_HD bool overrun() const { return pos * 8 - (uint64_t)cnt > len * 8; }
};

/* canonical decode of the next code (RFC 1951 3.2.2) from `bits` (LSB = first bit), lengths up to `maxlen`:
 * (length << 9) | symbol, or -1 if no code of at most maxlen bits matches */
template <int N>
MMI_HD int mmi_canonical(const mmi_huff<N> &h, uint32_t bits, int maxlen)
{
  int code = 0, first = 0, index = 0;
  for (int l = 1; l <= maxlen; l++) {
    code |= (int)(bits & 1);
    bits >>= 1;
    const int c = h.count[l];
    if (code < first + c) return (l << 9) | h.sym[index + code - first];
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

/* counts, canonical symbol order and (fast != nullptr) the lookup table of the code given by lens[0, n).
 * zlib's rules: an over-subscribed set is an error, an incomplete one is accepted only when its longest code has length
 * 1 (a single code), or when there is no code at all. Ends with the tables visible to every lane. */
template <int N>
MMI_HD int mmi_build(mmi_huff<N> &h, const uint8_t *lens, int n, uint16_t *fast, int lane, int nl)
{
  for (int l = lane; l < 16; l += nl) {
    int c = 0;
    for (int s = 0; s < n; s++) c += lens[s] == l;
    h.count[l] = (uint16_t)c;
  }
  mmi_sync();
  int left = 1, maxlen = 0;
  for (int l = 1; l < 16; l++) {
    left = (left << 1) - h.count[l];
    if (left < 0) return MMI_E_CODES;
    if (h.count[l]) maxlen = l;
  }
  if (left > 0 && maxlen > 1) return MMI_E_CODES;
  for (int l = lane; l < 16; l += nl) {
    if (l == 0) continue;
    int idx = 0;
    for (int j = 1; j < l; j++) idx += h.count[j];
    for (int s = 0; s < n; s++)
      if (lens[s] == l) h.sym[idx++] = (uint16_t)s;
  }
  mmi_sync();
  if (fast) {
    for (int e = lane; e < (1 << MMI_FAST); e += nl) {
      const int s = mmi_canonical(h, (uint32_t)e, MMI_FAST);
      fast[e] = s < 0 ? 0 : (uint16_t)s;
    }
    mmi_sync();
  }
  return MMI_OK;
}

/* next symbol of a literal/length or distance code; -1 if the bits are no code */
template <int N>
MMI_HD int mmi_decode(const mmi_huff<N> &h, const uint16_t *fast, mmi_bits &b)
{
  const uint32_t e = fast[b.buf & ((1u << MMI_FAST) - 1)];
  if (e) {
    b.take((int)(e >> 9));
    return (int)(e & 511);
  }
  const int s = mmi_canonical(h, (uint32_t)(b.buf & 0x7FFF), 15);
  if (s < 0) return s;
  b.take(s >> 9);
  return s & 511;
}

/* position of the i-th code-length code length in the header (RFC 1951 3.2.7: 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15) */
MMI_HD int mmi_clen_order(int i)
{
  /* 5 bits per entry, entries 0-11 and 12-18: a register constant instead of an array in local memory */
  return i < 12 ? (int)((0x22caa324e804a30ULL >> (5 * i)) & 31) : (int)((0x3c2e1346cULL >> (5 * (i - 12))) & 31);
}

/* decodes one raw DEFLATE stream: in[0, in_len) -> out[0, out_len); lanes 0..nl-1 of one warp call it together
 * (nl = 1 on the host). Returns an mmi_status, the same in every lane. */
MMI_HD int mmi_inflate(const uint8_t *in, uint64_t in_len, uint8_t *out, uint64_t out_len, mmi_tables &t, int lane, int nl)
{
  mmi_bits b{in, in_len, 0, 0, 0};
  uint64_t o = 0;
  int final = 0;
  while (!final) {
    b.refill();
    if (b.overrun()) return MMI_E_INPUT;
    final = (int)b.take(1);
    const int type = (int)b.take(2);
    if (type == 0) { /* stored */
      const uint64_t p0 = (b.pos * 8 - (uint64_t)b.cnt + 7) / 8;
      if (p0 + 4 > in_len) return MMI_E_INPUT;
      const uint32_t n = in[p0] | ((uint32_t)in[p0 + 1] << 8), nn = in[p0 + 2] | ((uint32_t)in[p0 + 3] << 8);
      if (n != (~nn & 0xFFFFu)) return MMI_E_STORED;
      const uint64_t p = p0 + 4;
      if (p + n > in_len) return MMI_E_INPUT;
      if (o + n > out_len) return MMI_E_OUTPUT;
      for (uint32_t k = (uint32_t)lane; k < n; k += (uint32_t)nl) out[o + k] = in[p + k];
      o += n;
      b.pos = p + n;
      b.buf = 0;
      b.cnt = 0;
      continue;
    }
    if (type == 3) return MMI_E_BTYPE;
    if (type == 1) { /* fixed codes: lengths 8/9/7/8 over 288 literal/length symbols, 5 over 32 distance symbols */
      for (int s = lane; s < 320; s += nl) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
      mmi_sync();
      if (int rc = mmi_build(t.lit, t.lens, 288, t.lfast, lane, nl)) return rc;
      if (int rc = mmi_build(t.dist, t.lens + 288, 32, t.dfast, lane, nl)) return rc;
    } else { /* dynamic codes */
      const int hlit = (int)b.take(5) + 257, hdist = (int)b.take(5) + 1, hclen = (int)b.take(4) + 4;
      if (hlit > 286 || hdist > 30) return MMI_E_CODES;
      uint8_t *cl = t.clens;
      b.refill();
      for (int i = 0; i < 19; i++) {
        const int v = i < hclen ? (int)b.take(3) : 0;
        if (i == 9) b.refill();
        if (lane == 0) cl[mmi_clen_order(i)] = (uint8_t)v;
      }
      mmi_sync();
      if (b.overrun()) return MMI_E_INPUT;
      if (int rc = mmi_build(t.clen, cl, 19, nullptr, lane, nl)) return rc;
      const int total = hlit + hdist;
      int i = 0;
      while (i < total) {
        b.refill();
        if (b.overrun()) return MMI_E_INPUT;
        const int e = mmi_canonical(t.clen, (uint32_t)(b.buf & 0x7F), 7);
        if (e < 0) return MMI_E_SYMBOL;
        b.take(e >> 9);
        const int s = e & 511;
        if (s < 16) {
          if (lane == 0) t.lens[i] = (uint8_t)s;
          i++;
          continue;
        }
        int v = 0, rep;
        if (s == 16) {
          if (i == 0) return MMI_E_CODES;
          mmi_sync();
          v = t.lens[i - 1];
          rep = 3 + (int)b.take(2);
        } else if (s == 17) {
          rep = 3 + (int)b.take(3);
        } else {
          rep = 11 + (int)b.take(7);
        }
        if (i + rep > total) return MMI_E_CODES;
        for (int r = lane; r < rep; r += nl) t.lens[i + r] = (uint8_t)v;
        i += rep;
      }
      mmi_sync();
      if (t.lens[256] == 0) return MMI_E_CODES;
      if (int rc = mmi_build(t.lit, t.lens, hlit, t.lfast, lane, nl)) return rc;
      if (int rc = mmi_build(t.dist, t.lens + hlit, hdist, t.dfast, lane, nl)) return rc;
    }
    /* literal/length and distance symbols until end-of-block; one refill covers the longest symbol pair (15+5+15+13 bits) */
    while (true) {
      b.refill();
      if (b.overrun()) return MMI_E_INPUT;
      const int s = mmi_decode(t.lit, t.lfast, b);
      if (s < 0) return MMI_E_SYMBOL;
      if (s < 256) {
        if (o >= out_len) return MMI_E_OUTPUT;
        if (lane == 0) out[o] = (uint8_t)s;
        o++;
        continue;
      }
      if (s == 256) break;
      const int li = s - 257;
      if (li > 28) return MMI_E_SYMBOL;
      int len;
      if (li < 8) len = 3 + li;
      else if (li == 28) len = 258;
      else {
        const int ex = (li >> 2) - 1;
        len = ((4 + (li & 3)) << ex) + 3 + (int)b.take(ex);
      }
      const int ds = mmi_decode(t.dist, t.dfast, b);
      if (ds < 0 || ds > 29) return MMI_E_SYMBOL;
      uint32_t dist;
      if (ds < 4) dist = (uint32_t)ds + 1;
      else {
        const int ex = (ds >> 1) - 1;
        dist = ((uint32_t)(2 + (ds & 1)) << ex) + 1 + b.take(ex);
      }
      if (b.overrun()) return MMI_E_INPUT;
      if (dist > o) return MMI_E_DIST;
      if ((uint64_t)len > out_len - o) return MMI_E_OUTPUT;
      /* out[o + k] = out[o + k - dist] repeats with period dist, so every byte can come from before o: no lane waits on
       * another inside one copy (distance < length included) */
      mmi_sync();
      const uint8_t *src = out + o - dist;
      for (int k = lane; k < len; k += nl) out[o + k] = src[(uint32_t)k < dist ? (uint32_t)k : (uint32_t)k % dist];
      o += (uint64_t)len;
    }
  }
  mmi_sync();
  const uint64_t end = (b.pos * 8 - (uint64_t)b.cnt + 7) / 8;
  if (end > in_len) return MMI_E_INPUT;
  if (end < in_len) return MMI_E_TRAILING;
  if (o != out_len) return MMI_E_SHORT;
  return MMI_OK;
}

/* ---- CRC-32 (RFC 1952 8), reflected polynomial 0xEDB88320 ---- */

MMI_HD void mmi_crc_table(uint32_t *tab, int lane, int nl)
{
  for (int i = lane; i < 256; i += nl) {
    uint32_t c = (uint32_t)i;
    for (int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    tab[i] = c;
  }
}

/* a * b modulo the CRC polynomial (bit 31 = x^0) */
MMI_HD uint32_t mmi_multmodp(uint32_t a, uint32_t b)
{
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
  }
  return p;
}

/* x^(8 n) modulo the polynomial: multiplying a CRC register by it appends n zero bytes */
MMI_HD uint32_t mmi_x8n(uint64_t n)
{
  uint32_t p = 1u << 31, sq = 1u << 23; /* x^0, x^8 */
  while (n) {
    if (n & 1) p = mmi_multmodp(sq, p);
    sq = mmi_multmodp(sq, sq);
    n >>= 1;
  }
  return p;
}

/* this lane's share of the CRC-32 of data[0, n): the lanes' shares XOR-ed together and passed to mmi_crc_finish give the
 * CRC. A lane takes one contiguous slice, runs the register from 0 over it and moves the result past the bytes after it. */
MMI_HD uint32_t mmi_crc_share(const uint32_t *tab, const uint8_t *data, uint64_t n, int lane, int nl)
{
  const uint64_t per = (n + (uint64_t)nl - 1) / (uint64_t)nl;
  const uint64_t lo = per * (uint64_t)lane < n ? per * (uint64_t)lane : n, hi = lo + per < n ? lo + per : n;
  uint32_t c = 0;
  for (uint64_t i = lo; i < hi; i++) c = tab[(c ^ data[i]) & 0xFF] ^ (c >> 8);
  return hi < n ? mmi_multmodp(mmi_x8n(n - hi), c) : c;
}

/* the register started at 0xFFFFFFFF is the register started at 0 plus 0xFFFFFFFF moved past all n bytes */
MMI_HD uint32_t mmi_crc_finish(uint32_t shares, uint64_t n) { return ~(shares ^ mmi_multmodp(mmi_x8n(n), 0xFFFFFFFFu)); }

#endif
