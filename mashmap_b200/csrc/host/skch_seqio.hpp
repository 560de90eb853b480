/*
 * skch_seqio.hpp -- FASTA / FASTQ (optionally gzip) reader.
 * Same observable behaviour as seqiter::for_each_seq_in_file (reference src/common/seqiter.hpp:20-111):
 * the record name is the header up to the first space (:82), sequence lines are concatenated, records
 * not matching keep_prefix / keep_seq are delivered with an empty sequence. Reads through zlib's gzFile
 * with a large buffer instead of the reference's 303-byte gzstream buffer (gzstream.h:50).
 */
#ifndef SKCH_SEQIO_HPP
#define SKCH_SEQIO_HPP

#include <cstdint>
#include <functional>
#include <string>
#include <unordered_set>
#include <vector>

namespace skch {
namespace seqio {

typedef std::function<void(const std::string &name, const std::string &seq)> SeqCallback;

/* returns false (after printing to stderr) if the file cannot be read or has an unknown format */
bool for_each_seq_in_file(const std::string &filename, const std::unordered_set<std::string> &keep_seq,
                          const std::string &keep_prefix, const SeqCallback &func);

/*
 * Bulk view of a plain (uncompressed) FASTA file: the file is mapped and cut into records by all host threads, so that
 * a caller can place the bases where it wants them (the pinned batch buffer) without going through one std::string per
 * record on one thread -- at tens of Gbp/s of mapping, a serial parser is the bottleneck of the program (SURVEY 8(f)-3).
 * Same record semantics as for_each_seq_in_file: a record starts at a line whose first byte is '>', its name is the
 * header up to the first space, its sequence is every following line up to the next record, concatenated (only the
 * '\n' bytes are dropped).
 */
struct FastaRecord {
  uint64_t name_off;  /* file offset of the first byte of the name */
  uint32_t name_len;
  uint64_t seq_off;   /* file offset of the first sequence line */
  uint64_t raw_len;   /* bytes from seq_off to the next record (or EOF), newlines included */
  uint64_t seq_len;   /* bases = raw_len minus the newlines */
};

/* the records of a FASTA text held in memory (a mapped file, or one window of an inflated BGZF file) */
class FastaText {
 public:
  /* cuts text[0, size) into records with up to `threads` host threads; text[0] is '>' and stays valid while in use */
  void parse(const char *text, uint64_t size, int threads);
  const std::vector<FastaRecord> &records() const { return recs_; }
  const char *data() const { return data_; }
  uint64_t size() const { return size_; }
  std::string name(const FastaRecord &r) const { return std::string(data_ + r.name_off, r.name_len); }
  /* copies the record's bases to dst (seq_len bytes) */
  void copy_bases(const FastaRecord &r, char *dst) const;
  /* the record's bases as nibbles (pack_bases below) to dst ((seq_len + 1) / 2 bytes), newlines dropped on the way */
  void pack_bases(const FastaRecord &r, uint8_t *dst) const;

 protected:
  const char *data_ = nullptr;
  uint64_t size_ = 0;
  std::vector<FastaRecord> recs_;
};

class FastaFile : public FastaText {
 public:
  FastaFile() = default;
  ~FastaFile();
  FastaFile(const FastaFile &) = delete;
  /* false if the file is not a plain FASTA file that can be mapped (gzip, FASTQ, pipe ...): use for_each_seq_in_file */
  bool open(const std::string &filename, int threads);

 private:
  int fd_ = -1;
};

/*
 * The one step of the BGZF reader that a caller chooses: inflate raw DEFLATE blocks, with mm_inflate_blocks' contract
 * (include/mashmap_b200.h). The program passes DeviceInflater; the tests pass HostInflater (the host build of
 * mm_inflate.h) or a fake. alloc / release give the reader's text buffers (pinned ones for the device).
 */
class BlockInflater {
 public:
  virtual ~BlockInflater() = default;
  /* 0, or nonzero with *bad_block = the failing block's index (or -1) and `error` saying why */
  virtual int inflate(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                      uint64_t n_blocks, uint8_t *out, int64_t *bad_block, std::string &error) = 0;
  virtual void *alloc(uint64_t bytes);
  virtual void release(void *p);
};

class HostInflater : public BlockInflater {
 public:
  int inflate(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
              uint64_t n_blocks, uint8_t *out, int64_t *bad_block, std::string &error) override;
};

class DeviceInflater : public BlockInflater {
 public:
  /* exits the program (status 1) if the device cannot be used */
  explicit DeviceInflater(int device);
  ~DeviceInflater() override;
  int inflate(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
              uint64_t n_blocks, uint8_t *out, int64_t *bad_block, std::string &error) override;
  void *alloc(uint64_t bytes) override;
  void release(void *p) override;

 private:
  void *inf_ = nullptr;
};

/*
 * FASTA in BGZF (bgzip) members, read window by window. A member is BGZF when its gzip header has FEXTRA with a 'BC'
 * subfield of length 2; its BSIZE, CRC32 and ISIZE place its data and its text before anything is inflated, so a
 * window's members go to the BlockInflater in one call. A member that is not BGZF, or one cut short by the end of the
 * file, is inflated on the host by zlib, in order, and bytes after the last member are ignored: the text is the one
 * gzread gives the line reader. A corrupt member is an error, where gzread would end the text early.
 */
class BgzfFasta {
 public:
  BgzfFasta() = default;
  ~BgzfFasta();
  BgzfFasta(const BgzfFasta &) = delete;
  /* false if the file cannot be mapped or its first member is not BGZF: the line reader handles it */
  bool open(const std::string &filename);
  /*
   * Inflates the text in windows of about window_bytes (grown while one record does not fit), cuts each window at its
   * last record start, carries the rest into the next window, and hands each window's records, parsed by `threads`
   * threads, to fn. Window i+1 is inflated while fn runs on window i. Returns 0; 1 if the text does not start with '>'
   * (nothing was handed over: the line reader handles the file); -1 on a corrupt member (error() names the file and the
   * member's byte offset).
   */
  int for_each_window(BlockInflater &inf, uint64_t window_bytes, int threads, const std::function<void(const FastaText &)> &fn);
  const std::string &error() const { return error_; }

 private:
  struct Buf { char *p = nullptr; uint64_t cap = 0, used = 0; };
  bool grow(BlockInflater &inf, Buf &b, uint64_t need);
  bool fill(BlockInflater &inf, Buf &b, uint64_t target);
  bool corrupt(uint64_t off, const std::string &why);

  std::string path_, error_;
  const uint8_t *d_ = nullptr;
  uint64_t size_ = 0, pos_ = 0;
  bool eof_ = false;
  int fd_ = -1;
  std::vector<uint8_t> stage_;
  std::vector<uint64_t> coff_, ooff_, moff_;
  std::vector<uint32_t> crc_;
};

/* text bytes per BGZF window for a run of --batchBases b: b, kept within [64 KiB, 256 MiB] */
uint64_t bgzf_window_bytes(uint64_t batch_bases);

/*
 * The device's input format (include/mashmap_b200.h, mm_map_segments_packed): one nibble per base, base i of the
 * sequence in byte i / 2 (low nibble first); nibble = 2-bit code (A 0, C 1, T 2, G 3: bits 1-2 of the upper-cased
 * letter) | 8 for every byte that is not ACGT after upper-casing -- makeUpperCaseAndValidDNA (reference
 * commonFunc.hpp:75-107) folded into the encoding. The parser touches every base once anyway; writing 4 bits instead of
 * 8 halves what crosses PCIe afterwards. dst gets (n + 1) / 2 bytes; an odd n leaves an 'N' nibble in the last byte.
 * AVX2 where the CPU has it (32 bases per step), plain C otherwise.
 */
void pack_bases(const char *src, uint64_t n, uint8_t *dst);

}  // namespace seqio
}  // namespace skch
#endif
