#include "skch_seqio.hpp"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include "../../../include/mashmap_b200.h"
#include "../mm_fastq.h"
#include "../mm_inflate.h"
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include <algorithm>
#include <atomic>
#include <cstring>
#include <iostream>
#include <memory>
#include <thread>
#include <vector>

namespace skch {
namespace seqio {

namespace {

class LineReader {
 public:
  explicit LineReader(const std::string &path) : buf_(1 << 20)
  {
    f_ = gzopen(path.c_str(), "rb");
    if (f_) gzbuffer(f_, 1 << 20);
  }
  ~LineReader() { if (f_) gzclose(f_); }
  bool ok() const { return f_ != nullptr; }
  /* std::getline semantics: false only when nothing could be read */
  bool getline(std::string &line)
  {
    line.clear();
    bool got = false;
    while (true) {
      if (pos_ == len_) {
        if (eof_) return got;
        int n = gzread(f_, buf_.data(), (unsigned)buf_.size());
        if (n <= 0) { eof_ = true; return got; }
        len_ = (size_t)n; pos_ = 0;
      }
      const char *b = buf_.data() + pos_;
      const char *nl = (const char *)memchr(b, '\n', len_ - pos_);
      if (nl) {
        line.append(b, nl - b);
        pos_ += (size_t)(nl - b) + 1;
        return true;
      }
      line.append(b, len_ - pos_);
      pos_ = len_;
      got = true;
    }
  }
  bool good() const { return !(eof_ && pos_ == len_); }

 private:
  gzFile f_ = nullptr;
  std::vector<char> buf_;
  size_t pos_ = 0, len_ = 0;
  bool eof_ = false;
};

}  // namespace

bool for_each_seq_in_file(const std::string &filename, const std::unordered_set<std::string> &keep_seq,
                          const std::string &keep_prefix, const SeqCallback &func)
{
  LineReader in(filename);
  if (!in.ok()) {
    std::cerr << "[mashmap-b200] ERROR: cannot open " << filename << std::endl;
    return false;
  }
  std::string line;
  in.getline(line);
  const bool is_fasta = !line.empty() && line[0] == '>';
  const bool is_fastq = !line.empty() && line[0] == '@';
  if (!is_fasta && !is_fastq) {
    std::cerr << "[mashmap-b200] unknown file format given to the sequence reader: " << filename << std::endl;
    return false;
  }
  auto wanted = [&](const std::string &name) {
    return (keep_prefix.empty() || name.compare(0, keep_prefix.length(), keep_prefix) == 0) &&
           (keep_seq.empty() || keep_seq.find(name) != keep_seq.end());
  };
  std::string seq;
  if (is_fasta) {
    bool more = true;
    while (more) {
      const std::string name = line.substr(1, line.find(' ') - 1); /* seqiter.hpp:82 */
      const bool keep = wanted(name);
      seq.clear();
      more = false;
      while (in.getline(line)) {
        if (!line.empty() && line[0] == '>') { more = true; break; }
        if (keep) seq.append(line);
      }
      func(name, seq);
    }
  } else {
    bool more = true;
    while (more) {
      const std::string name = line.substr(1, line.find(' ') - 1);
      const bool keep = wanted(name);
      std::string s, tmp;
      in.getline(s);
      in.getline(tmp);
      in.getline(tmp);
      more = in.getline(line) && !line.empty();
      func(name, keep ? s : std::string());
    }
  }
  return true;
}

/* ---- mapped FASTA ---- */

FastaFile::~FastaFile()
{
  if (data_) munmap((void *)data_, size_);
  if (fd_ >= 0) close(fd_);
}

bool FastaFile::open(const std::string &filename, int threads)
{
  fd_ = ::open(filename.c_str(), O_RDONLY);
  if (fd_ < 0) return false;
  struct stat st;
  if (fstat(fd_, &st) != 0 || !S_ISREG(st.st_mode) || st.st_size < 2) return false;
  size_ = (uint64_t)st.st_size;
  void *m = mmap(nullptr, size_, PROT_READ, MAP_PRIVATE, fd_, 0);
  if (m == MAP_FAILED) return false;
  data_ = (const char *)m;
  if (data_[0] != '>') return false; /* gzip magic, FASTQ, anything else: the line reader handles those */
  madvise(m, size_, MADV_SEQUENTIAL);
  parse(data_, size_, threads);
  return true;
}

void FastaText::parse(const char *text, uint64_t size, int threads)
{
  data_ = text;
  size_ = size;
  const int T = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)std::max(1, threads), size_ / (1 << 20) + 1));
  /* 1. record starts: '>' at the beginning of a line, found independently in T byte ranges */
  std::vector<std::vector<uint64_t>> starts((size_t)T);
  {
    std::vector<std::thread> pool;
    for (int t = 0; t < T; t++) {
      pool.emplace_back([&, t]() {
        const uint64_t lo = size_ * (uint64_t)t / (uint64_t)T, hi = size_ * (uint64_t)(t + 1) / (uint64_t)T;
        uint64_t p = lo;
        while (p < hi) {
          const char *q = (const char *)memchr(data_ + p, '>', hi - p);
          if (!q) break;
          p = (uint64_t)(q - data_);
          if (p == 0 || data_[p - 1] == '\n') starts[(size_t)t].push_back(p);
          p++;
        }
      });
    }
    for (auto &th : pool) th.join();
  }
  std::vector<uint64_t> all;
  for (auto &v : starts) all.insert(all.end(), v.begin(), v.end());
  /* 2. per record: header, sequence region, base count */
  recs_.assign(all.size(), FastaRecord{});
  {
    std::atomic<size_t> next{0};
    std::vector<std::thread> pool;
    for (int t = 0; t < T; t++) {
      pool.emplace_back([&]() {
        while (true) {
          const size_t b = next.fetch_add(4096);
          if (b >= all.size()) break;
          const size_t e = std::min(all.size(), b + 4096);
          for (size_t i = b; i < e; i++) {
            const uint64_t p = all[i], end = i + 1 < all.size() ? all[i + 1] : size_;
            const char *eol = (const char *)memchr(data_ + p, '\n', end - p);
            const uint64_t hdr_end = eol ? (uint64_t)(eol - data_) : end;
            const char *sp = (const char *)memchr(data_ + p + 1, ' ', hdr_end - (p + 1));
            FastaRecord &r = recs_[i];
            r.name_off = p + 1;
            r.name_len = (uint32_t)((sp ? (uint64_t)(sp - data_) : hdr_end) - (p + 1));
            r.seq_off = eol ? hdr_end + 1 : end;
            r.raw_len = end - r.seq_off;
            uint64_t nl = 0;
            for (const char *c = data_ + r.seq_off, *ce = data_ + end; c < ce;) {
              const char *q = (const char *)memchr(c, '\n', (size_t)(ce - c));
              if (!q) break;
              nl++;
              c = q + 1;
            }
            r.seq_len = r.raw_len - nl;
          }
        }
      });
    }
    for (auto &th : pool) th.join();
  }
}

void FastaText::copy_bases(const FastaRecord &r, char *dst) const
{
  const char *c = data_ + r.seq_off, *ce = c + r.raw_len;
  while (c < ce) {
    const char *q = (const char *)memchr(c, '\n', (size_t)(ce - c));
    const size_t n = (size_t)((q ? q : ce) - c);
    memcpy(dst, c, n);
    dst += n;
    c += n + 1;
  }
}

namespace {

struct NibTable {
  uint8_t t[256];
  NibTable()
  {
    for (int i = 0; i < 256; i++) t[i] = mmf_nib((uint8_t)i);
  }
};
const NibTable NIB;

void pack_scalar(const uint8_t *src, uint64_t n, uint8_t *dst)
{
  uint64_t i = 0;
  for (; i + 1 < n; i += 2) dst[i >> 1] = (uint8_t)(NIB.t[src[i]] | (NIB.t[src[i + 1]] << 4));
  if (i < n) dst[i >> 1] = (uint8_t)(NIB.t[src[i]] | 0x80);
}

#if defined(__x86_64__)
__attribute__((target("avx2"))) void pack_avx2(const uint8_t *src, uint64_t n, uint8_t *dst)
{
  const __m256i up = _mm256_set1_epi8((char)0xDF), three = _mm256_set1_epi8(3), eight = _mm256_set1_epi8(8);
  const __m256i cA = _mm256_set1_epi8('A'), cC = _mm256_set1_epi8('C'), cG = _mm256_set1_epi8('G'), cT = _mm256_set1_epi8('T');
  const __m256i mul = _mm256_set1_epi16(0x1001); /* low byte * 1 + high byte * 16 */
  uint64_t i = 0;
  for (; i + 32 <= n; i += 32) {
    const __m256i v = _mm256_loadu_si256((const __m256i *)(src + i));
    const __m256i x = _mm256_and_si256(v, up);
    const __m256i code = _mm256_and_si256(_mm256_srli_epi16(x, 1), three);
    const __m256i ok = _mm256_or_si256(_mm256_or_si256(_mm256_cmpeq_epi8(x, cA), _mm256_cmpeq_epi8(x, cC)),
                                       _mm256_or_si256(_mm256_cmpeq_epi8(x, cG), _mm256_cmpeq_epi8(x, cT)));
    const __m256i nib = _mm256_blendv_epi8(eight, code, ok);
    const __m256i w = _mm256_maddubs_epi16(nib, mul);                 /* 16 x (n0 + 16 n1) */
    const __m256i b = _mm256_packus_epi16(w, w);                      /* per 128-bit lane: 8 bytes, twice */
    const __m256i q = _mm256_permute4x64_epi64(b, 0x08);              /* lanes' low halves next to each other */
    _mm_storeu_si128((__m128i *)(dst + (i >> 1)), _mm256_castsi256_si128(q));
  }
  pack_scalar(src + i, n - i, dst + (i >> 1));
}
bool have_avx2()
{
  static const bool v = __builtin_cpu_supports("avx2");
  return v;
}
#endif

}  // namespace

void pack_bases(const char *src, uint64_t n, uint8_t *dst)
{
#if defined(__x86_64__)
  if (have_avx2()) { pack_avx2((const uint8_t *)src, n, dst); return; }
#endif
  pack_scalar((const uint8_t *)src, n, dst);
}

void FastaText::pack_bases(const FastaRecord &r, uint8_t *dst) const
{
  /* lines are gathered into an even-sized stretch of text first (a line may have an odd length; nibble pairs must not
   * straddle two pack calls), then packed: the stretch stays in the L1/L2 cache */
  char buf[8192 + 64];
  size_t fill = 0;
  const char *c = data_ + r.seq_off, *ce = c + r.raw_len;
  while (c < ce) {
    const char *q = (const char *)memchr(c, '\n', (size_t)(ce - c));
    size_t n = (size_t)((q ? q : ce) - c);
    const char *next = c + n + 1;
    while (n) {
      const size_t take = std::min(n, (size_t)8192 - fill);
      memcpy(buf + fill, c, take);
      fill += take; c += take; n -= take;
      if (fill == 8192) { seqio::pack_bases(buf, fill, dst); dst += fill / 2; fill = 0; }
    }
    c = next;
  }
  if (fill) seqio::pack_bases(buf, fill, dst);
}

/* ---- BGZF ---- */

void *BlockInflater::alloc(uint64_t bytes) { return malloc(bytes); }
void BlockInflater::release(void *p) { free(p); }

int HostInflater::inflate(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                          uint64_t n_blocks, uint8_t *out, int64_t *bad_block, std::string &error)
{
  static const struct CrcTab {
    uint32_t t[256];
    CrcTab() { mmi_crc_table(t, 0, 1); }
  } tab;
  std::unique_ptr<mmi_tables> t(new mmi_tables());
  *bad_block = -1;
  for (uint64_t i = 0; i < n_blocks; i++) {
    const uint64_t on = out_off[i + 1] - out_off[i];
    int rc = mmi_inflate(comp + comp_off[i], comp_off[i + 1] - comp_off[i], out + out_off[i], on, *t, 0, 1);
    if (rc == MMI_OK && mmi_crc_finish(mmi_crc_share(tab.t, out + out_off[i], on, 0, 1), on) != crc[i]) rc = MMI_E_CRC;
    if (rc != MMI_OK) {
      *bad_block = (int64_t)i;
      error = "inflate status " + std::to_string(rc);
      return rc;
    }
  }
  return 0;
}

DeviceInflater::DeviceInflater(int device)
{
  mm_inflater *h = nullptr;
  if (mm_inflater_create(device, &h) != MM_OK) {
    std::cerr << "[mashmap-b200] ERROR: mm_inflater_create: " << mm_inflater_error(nullptr) << std::endl;
    exit(1);
  }
  inf_ = h;
}

DeviceInflater::~DeviceInflater() { mm_inflater_destroy((mm_inflater *)inf_); }

int DeviceInflater::inflate(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                            uint64_t n_blocks, uint8_t *out, int64_t *bad_block, std::string &error)
{
  const int rc = mm_inflate_blocks((mm_inflater *)inf_, comp, comp_off, out_off, crc, n_blocks, out, bad_block);
  if (rc != MM_OK) error = mm_inflater_error((mm_inflater *)inf_);
  return rc;
}

void *DeviceInflater::alloc(uint64_t bytes)
{
  void *p = nullptr;
  return mm_host_alloc(&p, bytes) == MM_OK ? p : nullptr;
}

void DeviceInflater::release(void *p) { mm_host_free(p); }

uint64_t bgzf_window_bytes(uint64_t batch_bases) { return std::min<uint64_t>(std::max<uint64_t>(batch_bases, 1 << 16), 1ULL << 28); }

uint64_t fastq_window_bytes(uint64_t batch_bases)
{
  return std::min<uint64_t>(std::max<uint64_t>(2 * std::min<uint64_t>(batch_bases, 1ULL << 40), 1 << 16), 1ULL << 29);
}

namespace {

inline uint32_t le16(const uint8_t *p) { return p[0] | ((uint32_t)p[1] << 8); }
inline uint32_t le32(const uint8_t *p) { return le16(p) | (le16(p + 2) << 16); }

struct Member {
  uint64_t data_off, data_len, next;
  uint32_t crc, isize;
};

/* 1: a complete BGZF member at p; 0: a gzip member for zlib (not BGZF, unusual header, or cut short); -1: no member
 * starts at p (end of file, or trailing bytes that gzread ignores) */
int scan_member(const uint8_t *d, uint64_t size, uint64_t p, Member &m)
{
  if (size - p < 2 || d[p] != 0x1F || d[p + 1] != 0x8B) return -1;
  if (size - p < 12 || d[p + 2] != 8 || d[p + 3] != 4) return 0; /* FEXTRA alone: BGZF sets no other flag */
  const uint64_t xlen = le16(d + p + 10), x0 = p + 12, x1 = x0 + xlen;
  if (x1 > size) return 0;
  uint64_t bsize = 0;
  bool bc = false;
  for (uint64_t q = x0; q + 4 <= x1;) {
    const uint64_t slen = le16(d + q + 2);
    if (d[q] == 'B' && d[q + 1] == 'C' && slen == 2 && q + 6 <= x1) { bsize = le16(d + q + 4); bc = true; }
    q += 4 + slen;
  }
  const uint64_t total = bsize + 1;
  if (!bc || total < 12 + xlen + 8 || p + total > size) return 0;
  m.data_off = x1;
  m.data_len = p + total - 8 - x1;
  m.crc = le32(d + p + total - 8);
  m.isize = le32(d + p + total - 4);
  m.next = p + total;
  return m.isize <= 65536 ? 1 : 0; /* BGZF blocks hold at most 64 KiB of text; zlib takes anything else */
}

}  // namespace

BgzfMembers::~BgzfMembers()
{
  if (d_) munmap((void *)d_, size_);
  if (fd_ >= 0) close(fd_);
}

bool BgzfMembers::open(const std::string &filename)
{
  path_ = filename;
  fd_ = ::open(filename.c_str(), O_RDONLY);
  if (fd_ < 0) return false;
  struct stat st;
  if (fstat(fd_, &st) != 0 || !S_ISREG(st.st_mode) || st.st_size < 18) return false;
  size_ = (uint64_t)st.st_size;
  void *m = mmap(nullptr, size_, PROT_READ, MAP_PRIVATE, fd_, 0);
  if (m == MAP_FAILED) { size_ = 0; return false; }
  d_ = (const uint8_t *)m;
  madvise(m, size_, MADV_SEQUENTIAL);
  Member mb;
  return scan_member(d_, size_, 0, mb) == 1;
}

bool BgzfMembers::corrupt(uint64_t off, const std::string &why, std::string &error)
{
  error = "[mashmap-b200] ERROR: " + path_ + ": corrupt gzip/BGZF block at byte offset " + std::to_string(off) + ": " + why;
  return false;
}

bool BgzfMembers::next(uint64_t want, const BlocksFn &blocks, const TextFn &text, std::string &error)
{
  uint64_t sent = 0;
  while (sent < want && !eof_) {
    Member m;
    const int kind = scan_member(d_, size_, pos_, m);
    if (kind < 0) { eof_ = true; break; }
    if (kind == 0) { /* one gzip member through zlib, as gzread would inflate it */
      z_stream zs;
      memset(&zs, 0, sizeof zs);
      if (inflateInit2(&zs, 15 + 16) != Z_OK) return corrupt(pos_, "zlib cannot start", error);
      const uint64_t start = pos_;
      uint64_t in_left = size_ - pos_;
      const uint8_t *in = d_ + pos_;
      int rc = Z_OK;
      chunk_.resize(1 << 20);
      while (true) {
        zs.next_out = (Bytef *)chunk_.data();
        zs.avail_out = (uInt)chunk_.size();
        const uInt feed = (uInt)std::min<uint64_t>(in_left, 1u << 30);
        zs.next_in = (Bytef *)in;
        zs.avail_in = feed;
        rc = inflate(&zs, Z_NO_FLUSH);
        const uint64_t got = chunk_.size() - zs.avail_out;
        in += feed - zs.avail_in;
        in_left -= feed - zs.avail_in;
        if (got && !text(chunk_.data(), got, error)) { inflateEnd(&zs); return false; }
        sent += got;
        if (rc == Z_STREAM_END) break;
        if (rc == Z_BUF_ERROR && in_left == 0) break; /* cut short: gzread hands over what inflated, then ends */
        if (rc != Z_OK && rc != Z_BUF_ERROR) break;
        if (in_left == 0 && zs.avail_out != 0) { rc = Z_BUF_ERROR; break; }
      }
      const char *msg = zs.msg;
      inflateEnd(&zs);
      if (rc == Z_STREAM_END) pos_ = (uint64_t)(in - d_);
      else if (rc == Z_BUF_ERROR) eof_ = true;
      else return corrupt(start, msg ? msg : "zlib error", error);
      continue;
    }
    /* consecutive BGZF members up to `want`, at least one: one call of the inflater */
    coff_.assign(1, 0);
    ooff_.assign(1, 0);
    moff_.clear();
    crc_.clear();
    uint64_t p = pos_, out = 0;
    while (true) {
      moff_.push_back(p);
      crc_.push_back(m.crc);
      coff_.push_back(coff_.back() + m.data_len);
      out += m.isize;
      ooff_.push_back(out);
      p = m.next;
      if (sent + out >= want || scan_member(d_, size_, p, m) != 1) break;
    }
    stage_.resize(coff_.back());
    for (size_t i = 0; i < moff_.size(); i++) {
      Member mi;
      scan_member(d_, size_, moff_[i], mi);
      memcpy(stage_.data() + coff_[i], d_ + mi.data_off, mi.data_len);
    }
    int64_t bad = -1;
    std::string why;
    const int rc = blocks(stage_.data(), coff_.data(), ooff_.data(), crc_.data(), moff_.size(), &bad, why, error);
    if (rc < 0) return false;
    if (rc != 0) return corrupt(bad >= 0 && (size_t)bad < moff_.size() ? moff_[(size_t)bad] : pos_, why, error);
    sent += out;
    pos_ = p;
  }
  return true;
}

bool BgzfFasta::grow(BlockInflater &inf, Buf &b, uint64_t need, std::string &error)
{
  if (need <= b.cap) return true;
  const uint64_t cap = std::max<uint64_t>(need, b.cap + b.cap / 2);
  char *q = (char *)inf.alloc(cap);
  if (!q) {
    error = "[mashmap-b200] ERROR: cannot allocate " + std::to_string(cap) + " bytes of host memory to read " + mem_.path();
    return false;
  }
  if (b.used) memcpy(q, b.p, b.used);
  if (b.p) inf.release(b.p);
  b.p = q;
  b.cap = cap;
  return true;
}

/* appends text to b until it holds `target` bytes or the members end */
bool BgzfFasta::fill(BlockInflater &inf, Buf &b, uint64_t target, std::string &error)
{
  if (b.used >= target) return true;
  return mem_.next(
      target - b.used,
      [&](const uint8_t *comp, const uint64_t *coff, const uint64_t *ooff, const uint32_t *crc, uint64_t n, int64_t *bad,
          std::string &why, std::string &err) {
        if (!grow(inf, b, b.used + ooff[n] + 1, err)) return -1;
        const int rc = inf.inflate(comp, coff, ooff, crc, n, (uint8_t *)b.p + b.used, bad, why);
        if (rc == 0) b.used += ooff[n];
        return rc == 0 ? 0 : 1;
      },
      [&](const uint8_t *t, uint64_t n, std::string &err) {
        if (!grow(inf, b, b.used + n, err)) return false;
        memcpy(b.p + b.used, t, n);
        b.used += n;
        return true;
      },
      error);
}

int BgzfFasta::for_each_window(BlockInflater &inf, uint64_t window_bytes, int threads, const std::function<void(const FastaText &)> &fn)
{
  Buf cur, nxt;
  struct Release {
    BlockInflater &inf;
    Buf &a, &b;
    ~Release() { if (a.p) inf.release(a.p); if (b.p) inf.release(b.p); }
  } release{inf, cur, nxt};
  window_bytes = std::max<uint64_t>(window_bytes, 1);
  if (!fill(inf, cur, window_bytes, error_)) return -1;
  if (cur.used == 0 || cur.p[0] != '>') return 1;
  FastaText text;
  while (cur.used) {
    /* cut after the last record start that is not the window's first byte; a record longer than the window grows it */
    uint64_t cut = cur.used;
    if (!mem_.at_end()) {
      cut = 0;
      for (uint64_t q = cur.used; q > 1;) {
        const char *g = (const char *)memrchr(cur.p + 1, '>', q - 1);
        if (!g) break;
        if (g[-1] == '\n') { cut = (uint64_t)(g - cur.p); break; }
        q = (uint64_t)(g - cur.p);
      }
      if (cut == 0) {
        if (!fill(inf, cur, cur.used + window_bytes, error_)) return -1;
        continue;
      }
    }
    const uint64_t carry = cur.used - cut;
    if (!grow(inf, nxt, carry + window_bytes + 1, error_)) return -1;
    memcpy(nxt.p, cur.p + cut, carry);
    nxt.used = carry;
    bool ok = true;
    std::string err;
    std::thread next;
    if (!mem_.at_end()) next = std::thread([&]() { ok = fill(inf, nxt, carry + window_bytes, err); });
    text.parse(cur.p, cut, threads);
    fn(text);
    if (next.joinable()) next.join();
    if (!ok) { error_ = err; return -1; }
    std::swap(cur, nxt);
    nxt.used = 0;
  }
  return 0;
}

/* ---- FASTQ ---- */

void *FastqParser::alloc(uint64_t bytes) { return malloc(bytes); }
void FastqParser::release(void *p) { free(p); }

int HostFastqParser::append_text(const uint8_t *text, uint64_t n, std::string &)
{
  win_.insert(win_.end(), text, text + n);
  return 0;
}

int HostFastqParser::append_blocks(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                                   uint64_t n_blocks, int64_t *bad_block, std::string &error)
{
  const uint64_t at = win_.size();
  win_.resize(at + out_off[n_blocks] - out_off[0]);
  HostInflater inf;
  const int rc = inf.inflate(comp, comp_off, out_off, crc, n_blocks, win_.data() + at - out_off[0], bad_block, error);
  if (rc != 0) win_.resize(at);
  return rc;
}

/* the host build of mm_fastq_cut: the same statement (mm_fastq.h) with one lane */
int HostFastqParser::cut(int last, mm_fastq_records &res, std::string &)
{
  const uint8_t *text = win_.data();
  const uint64_t n = win_.size();
  nl_.clear();
  for (uint64_t p = 0; p < n; p += 4)
    for (uint32_t w = mmf_newline_mask(mmf_word(text, n, p)); w; w &= w - 1) nl_.push_back(p + (uint64_t)(__builtin_ctz(w) >> 3));
  const uint64_t N = nl_.size();
  uint64_t first_empty = mmf_empty_header_after(text, n, ~0ULL, ~0ULL);
  for (uint64_t j = 0; j < N; j++) first_empty = std::min(first_empty, mmf_empty_header_after(text, n, j, nl_[j]));
  uint64_t consumed = 0;
  int ended = 0;
  const uint64_t R = mmf_extent(nl_.data(), N, n, last, first_empty, &consumed, &ended);
  Out &o = out_[next_];
  next_ ^= 1;
  o.name_off.assign(1, 0);
  o.nib_off.assign(1, 0);
  o.seq_len.clear();
  o.names.clear();
  o.nibbles.clear();
  for (uint64_t r = 0; r < R; r++) {
    const mmf_record f = mmf_fields(text, n, nl_.data(), N, r);
    o.names.append((const char *)text + f.name, f.name_len);
    for (uint64_t k = 0; k < (f.seq_len + 1) / 2; k++) o.nibbles.push_back(mmf_nib_byte(text + f.seq, f.seq_len, k));
    o.name_off.push_back(o.names.size());
    o.nib_off.push_back(o.nibbles.size());
    o.seq_len.push_back(f.seq_len);
  }
  res.n_records = R;
  res.name_off = o.name_off.data();
  res.nib_off = o.nib_off.data();
  res.seq_len = o.seq_len.data();
  res.names = o.names.data();
  res.nibbles = o.nibbles.data();
  res.consumed = consumed;
  res.ended = ended;
  win_.erase(win_.begin(), win_.begin() + (ptrdiff_t)consumed);
  return 0;
}

DeviceFastqParser::DeviceFastqParser(int device)
{
  if (mm_fastq_create(device, &fq_) != MM_OK) {
    std::cerr << "[mashmap-b200] ERROR: mm_fastq_create: " << mm_fastq_error(nullptr) << std::endl;
    exit(1);
  }
}

DeviceFastqParser::~DeviceFastqParser() { mm_fastq_destroy(fq_); }

int DeviceFastqParser::append_text(const uint8_t *text, uint64_t n, std::string &error)
{
  const int rc = mm_fastq_append_text(fq_, text, n);
  if (rc != MM_OK) error = mm_fastq_error(fq_);
  return rc;
}

int DeviceFastqParser::append_blocks(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                                     uint64_t n_blocks, int64_t *bad_block, std::string &error)
{
  const int rc = mm_fastq_append_blocks(fq_, comp, comp_off, out_off, crc, n_blocks, bad_block);
  if (rc != MM_OK) error = mm_fastq_error(fq_);
  return rc;
}

int DeviceFastqParser::cut(int last, mm_fastq_records &out, std::string &error)
{
  const int rc = mm_fastq_cut(fq_, last, &out);
  if (rc != MM_OK) error = mm_fastq_error(fq_);
  return rc;
}

void *DeviceFastqParser::alloc(uint64_t bytes)
{
  void *p = nullptr;
  return mm_host_alloc(&p, bytes) == MM_OK ? p : nullptr;
}

void DeviceFastqParser::release(void *p) { mm_host_free(p); }

FastqReader::~FastqReader()
{
  if (d_) munmap((void *)d_, size_);
  if (fd_ >= 0) close(fd_);
}

bool FastqReader::open(const std::string &filename)
{
  path_ = filename;
  fd_ = ::open(filename.c_str(), O_RDONLY);
  if (fd_ < 0) return false;
  struct stat st;
  if (fstat(fd_, &st) != 0 || !S_ISREG(st.st_mode) || st.st_size < 1) return false;
  char first = 0;
  if (pread(fd_, &first, 1, 0) != 1) return false;
  if (first == '@') {
    size_ = (uint64_t)st.st_size;
    void *m = mmap(nullptr, size_, PROT_READ, MAP_PRIVATE, fd_, 0);
    if (m == MAP_FAILED) { size_ = 0; return false; }
    d_ = (const uint8_t *)m;
    madvise(m, size_, MADV_SEQUENTIAL);
    return true;
  }
  if (!mem_.open(filename)) return false;
  /* the first byte of the text, as the line reader sees it */
  gzFile f = gzopen(filename.c_str(), "rb");
  if (!f) return false;
  const int got = gzread(f, &first, 1);
  gzclose(f);
  bgzf_ = got == 1 && first == '@';
  return bgzf_;
}

/* appends text to the parser's window until it holds `target` bytes or the input ends */
bool FastqReader::load(FastqParser &p, uint64_t target, int threads)
{
  std::string why;
  if (bgzf_) {
    if (held_ >= target) return true;
    return mem_.next(
        target - held_,
        [&](const uint8_t *comp, const uint64_t *coff, const uint64_t *ooff, const uint32_t *crc, uint64_t n, int64_t *bad,
            std::string &w, std::string &) {
          const int rc = p.append_blocks(comp, coff, ooff, crc, n, bad, w);
          if (rc == 0) held_ += ooff[n];
          return rc == 0 ? 0 : 1;
        },
        [&](const uint8_t *t, uint64_t n, std::string &err) {
          if (p.append_text(t, n, why) == 0) { held_ += n; return true; }
          err = "[mashmap-b200] ERROR: " + path_ + ": " + why;
          return false;
        },
        error_);
  }
  while (held_ < target && pos_ < size_) {
    const uint64_t n = std::min(target - held_, size_ - pos_);
    const uint64_t chunk = std::min<uint64_t>(n, 1ULL << 28);
    if (chunk > stage_cap_) {
      if (stage_) p.release(stage_);
      stage_cap_ = std::max(chunk, std::min<uint64_t>(target, 1ULL << 28));
      stage_ = (uint8_t *)p.alloc(stage_cap_);
      if (!stage_) {
        stage_cap_ = 0;
        error_ = "[mashmap-b200] ERROR: cannot allocate " + std::to_string(chunk) + " bytes of host memory to read " + path_;
        return false;
      }
    }
    /* the mapped file into the pinned stage, by all host threads (the page faults of the mapping are most of the cost) */
    const int T = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)std::max(1, threads), chunk / (1 << 20) + 1));
    auto copy = [&](int t) {
      const uint64_t lo = chunk * (uint64_t)t / (uint64_t)T, hi = chunk * (uint64_t)(t + 1) / (uint64_t)T;
      memcpy(stage_ + lo, d_ + pos_ + lo, hi - lo);
    };
    if (T == 1) copy(0);
    else {
      std::vector<std::thread> pool;
      for (int t = 0; t < T; t++) pool.emplace_back(copy, t);
      for (auto &th : pool) th.join();
    }
    if (p.append_text(stage_, chunk, why) != 0) {
      error_ = "[mashmap-b200] ERROR: " + path_ + ": " + why;
      return false;
    }
    pos_ += chunk;
    held_ += chunk;
  }
  return true;
}

int FastqReader::for_each_window(FastqParser &p, uint64_t window_bytes, int threads, const std::function<void(const mm_fastq_records &)> &fn)
{
  window_bytes = std::max<uint64_t>(window_bytes, 1);
  struct Release {
    FastqParser &p;
    uint8_t *&stage;
    uint64_t &cap;
    ~Release() { if (stage) p.release(stage); stage = nullptr; cap = 0; }
  } release{p, stage_, stage_cap_};
  struct Cut { mm_fastq_records rec; bool done = false; };
  /* appends and cuts until a cut returns records or the file ends (a record larger than the window grows it), or after
   * one cut when `once`: a cut's results last until the cut after next, so only one cut may run while fn reads */
  auto step = [&](Cut &c, bool once) {
    uint64_t target = held_ + window_bytes;
    while (true) {
      if (!load(p, target, threads)) return false;
      const int last = at_end() ? 1 : 0;
      std::string why;
      if (p.cut(last, c.rec, why) != 0) {
        error_ = "[mashmap-b200] ERROR: " + path_ + ": " + why;
        return false;
      }
      held_ -= c.rec.consumed;
      c.done = last || c.rec.ended;
      if (c.rec.n_records || c.done || once) return true;
      target = std::max(held_ + window_bytes, 2 * held_);
    }
  };
  Cut cur;
  if (!step(cur, false)) return -1;
  while (true) {
    Cut nxt;
    bool ok = true;
    std::thread th;
    if (!cur.done) th = std::thread([&]() { ok = step(nxt, true); });
    if (cur.rec.n_records) fn(cur.rec);
    if (th.joinable()) th.join();
    if (!ok) return -1;
    if (cur.done) return 0;
    if (!nxt.rec.n_records && !nxt.done && !step(nxt, false)) return -1;
    cur = nxt;
  }
}

}  // namespace seqio
}  // namespace skch
