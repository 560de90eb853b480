/*
 * mm_fastq.h -- where a FASTQ text's records are, and their bases as nibbles.
 *
 * One statement, compiled __host__ __device__ like mm_inflate.h: the kernels in mm_fastq.cu run it over a window of
 * text in device memory, the host (skch::seqio's host parser, the tests) with one lane.
 *
 * The records are the line reader's (skch_seqio.cpp, for_each_seq_in_file; reference seqiter.hpp:98-110): strictly
 * four lines per record -- header, sequence, '+' line, quality line -- and nothing after the first byte of the file is
 * checked for '@' or '+'. So line L is a header iff L % 4 == 0, and where records start follows from counting newlines
 * alone: a prefix sum, no resynchronisation heuristic. In detail:
 *  - a line ends at its '\n' (not included) or at the end of the text; a line that would start at the end of the text
 *    does not exist;
 *  - the name is the header from its byte 1 up to the first ' ' (std::string::find(' ')); a header whose byte 0 is ' '
 *    gives the whole rest of the line (find returns 0, and substr(1, npos) follows);
 *  - the sequence is the second line exactly as written ('\r' included); empty when that line does not exist;
 *  - an empty line in header position ends the file: nothing after it is read;
 *  - a record cut short by the end of the file after one, two or three lines is still a record.
 */
#ifndef MM_FASTQ_H
#define MM_FASTQ_H

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define MMF_HD __host__ __device__ __forceinline__
#else
#define MMF_HD inline
#endif

enum mmf_line { MMF_HEADER = 0, MMF_SEQ = 1, MMF_PLUS = 2, MMF_QUAL = 3 };

#define MMF_NONE (~0ULL) /* no empty header line */

MMF_HD int mmf_line_kind(uint64_t line) { return (int)(line & 3); }

MMF_HD int mmf_popc(uint32_t x)
{
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}

/* 0x80 in each byte of the little-endian word w that is '\n', 0 elsewhere (exact: no borrow between bytes) */
MMF_HD uint32_t mmf_newline_mask(uint32_t w)
{
  const uint32_t x = w ^ 0x0A0A0A0Au;
  return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);
}

/* the word of text[pos, pos + 4), bytes at or past n read as 0 (not '\n'); pos is a multiple of 4 */
MMF_HD uint32_t mmf_word(const uint8_t *text, uint64_t n, uint64_t pos)
{
  if (pos + 4 <= n) {
#if defined(__CUDA_ARCH__)
    return *(const uint32_t *)(text + pos);
#else
    uint32_t w;
    memcpy(&w, text + pos, 4);
    return w;
#endif
  }
  uint32_t w = 0;
  for (uint64_t i = pos; i < n && i < pos + 4; i++) w |= (uint32_t)text[i] << (8 * (i - pos));
  return w;
}

/* newlines in text[pos, pos + bytes) (pos and bytes multiples of 4), the part at or past n counting none: one tile's
 * count, or one thread's share of it */
MMF_HD uint32_t mmf_count_newlines(const uint8_t *text, uint64_t n, uint64_t pos, uint64_t bytes)
{
  uint32_t c = 0;
  for (uint64_t p = pos; p < pos + bytes && p < n; p += 4) c += (uint32_t)mmf_popc(mmf_newline_mask(mmf_word(text, n, p)));
  return c;
}

/* where line `line` starts in text[0, n) whose N newlines are at nl[0, N): n if it does not exist */
MMF_HD uint64_t mmf_line_start(const uint64_t *nl, uint64_t N, uint64_t n, uint64_t line)
{
  return line == 0 ? 0 : line - 1 < N ? nl[line - 1] + 1 : n;
}

/* where line `line` ends: its '\n', or n */
MMF_HD uint64_t mmf_line_end(const uint64_t *nl, uint64_t N, uint64_t n, uint64_t line) { return line < N ? nl[line] : n; }

/* the record index whose header line starts right after newline j (at byte p) and is empty, else MMF_NONE; the
 * window's first line (a header) is checked with j = ~0, p = ~0 */
MMF_HD uint64_t mmf_empty_header_after(const uint8_t *text, uint64_t n, uint64_t j, uint64_t p)
{
  const uint64_t line = j + 1, start = p + 1;
  if (mmf_line_kind(line) != MMF_HEADER || start >= n || text[start] != '\n') return MMF_NONE;
  return line / 4;
}

/*
 * How many records a cut of text[0, n) returns, and how many bytes it takes. first_empty is the least record index
 * whose header line is empty (MMF_NONE if none). An empty header ends the file: the records before it, all the text
 * taken, *ended = 1. Otherwise with last = 1 (the end of the file) every record whose header starts inside the text,
 * all the text taken; with last = 0 the records whose fourth line ends inside the text, and the text up to the next
 * header (the rest is the start of a record, kept for the next cut).
 */
MMF_HD uint64_t mmf_extent(const uint64_t *nl, uint64_t N, uint64_t n, int last, uint64_t first_empty, uint64_t *consumed,
                           int *ended)
{
  *ended = first_empty != MMF_NONE;
  if (*ended) {
    *consumed = n;
    return first_empty;
  }
  if (last) {
    uint64_t R = N / 4 + 1;
    if (mmf_line_start(nl, N, n, 4 * (R - 1)) >= n) R--;
    *consumed = n;
    return R;
  }
  const uint64_t R = N / 4;
  *consumed = R ? mmf_line_start(nl, N, n, 4 * R) : 0;
  return R;
}

struct mmf_record {
  uint64_t name;     /* first byte of the name (the header's byte 1) */
  uint64_t name_len;
  uint64_t seq;      /* first byte of the sequence line (n when there is none) */
  uint64_t seq_len;
};

/* record r of text[0, n), one that mmf_extent returns (its header line exists and is not empty) */
MMF_HD mmf_record mmf_fields(const uint8_t *text, uint64_t n, const uint64_t *nl, uint64_t N, uint64_t r)
{
  const uint64_t hdr = mmf_line_start(nl, N, n, 4 * r), he = mmf_line_end(nl, N, n, 4 * r);
  mmf_record f;
  f.name = hdr + 1;
  uint64_t e = he;
  if (text[hdr] != ' ')
    for (uint64_t q = f.name; q < he; q++)
      if (text[q] == ' ') { e = q; break; }
  f.name_len = e - f.name;
  f.seq = mmf_line_start(nl, N, n, 4 * r + 1);
  f.seq_len = mmf_line_end(nl, N, n, 4 * r + 1) - f.seq;
  return f;
}

/* the nibble of one base: seqio::pack_bases' encoding (2-bit code of A C T G in either case, 8 for anything else) */
MMF_HD uint8_t mmf_nib(uint8_t c)
{
  const uint8_t u = c & 0xDF;
  return u == 'A' ? 0 : u == 'C' ? 1 : u == 'T' ? 2 : u == 'G' ? 3 : 8;
}

/* byte k of the nibbles of the sequence s[0, len): bases 2k (low nibble) and 2k + 1, an 'N' nibble past the end */
MMF_HD uint8_t mmf_nib_byte(const uint8_t *s, uint64_t len, uint64_t k)
{
  const uint64_t i = 2 * k;
  return (uint8_t)(mmf_nib(s[i]) | ((i + 1 < len ? mmf_nib(s[i + 1]) : 8) << 4));
}

/* the index i in [0, n) with off[i] <= x < off[i + 1], for non-decreasing off[0, n] with off[0] <= x < off[n] */
MMF_HD uint64_t mmf_find(const uint64_t *off, uint64_t n, uint64_t x)
{
  uint64_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (off[mid] <= x) lo = mid;
    else hi = mid;
  }
  return lo;
}

#endif
