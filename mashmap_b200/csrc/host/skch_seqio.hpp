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

#include "../../../include/mashmap_b200.h"

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
 * The gzip members of a BGZF file, walked in order. A member is BGZF when its gzip header has FEXTRA with a 'BC'
 * subfield of length 2; its BSIZE, CRC32 and ISIZE place its data and its text before anything is inflated, so a run of
 * BGZF members goes to the caller's inflater in one call. A member that is not BGZF, or one cut short by the end of the
 * file, is inflated on the host by zlib, in order, and bytes after the last member are ignored: the text is the one
 * gzread gives the line reader. A corrupt member is an error, where gzread would end the text early.
 */
class BgzfMembers {
 public:
  BgzfMembers() = default;
  ~BgzfMembers();
  BgzfMembers(const BgzfMembers &) = delete;
  /* false if the file cannot be mapped or its first member is not BGZF */
  bool open(const std::string &filename);
  bool at_end() const { return eof_; }
  const std::string &path() const { return path_; }
  /* a run of BGZF members: mm_inflate_blocks' arguments (ooff[0] = 0, ooff[n] = its text bytes); 0, or nonzero with
   * *bad_block = the failing member's index in the run (or -1) and `why`; a negative return means the callee set
   * `error` itself (not a corrupt member) */
  typedef std::function<int(const uint8_t *comp, const uint64_t *coff, const uint64_t *ooff, const uint32_t *crc, uint64_t n,
                            int64_t *bad_block, std::string &why, std::string &error)> BlocksFn;
  /* text that zlib inflated on the host; false if the callee set `error` */
  typedef std::function<bool(const uint8_t *text, uint64_t n, std::string &error)> TextFn;
  /* hands the members' text on, in order, until `want` bytes went out or the members end; false on an error (a corrupt
   * member: `error` names the file and the member's byte offset) */
  bool next(uint64_t want, const BlocksFn &blocks, const TextFn &text, std::string &error);

 private:
  bool corrupt(uint64_t off, const std::string &why, std::string &error);

  std::string path_;
  const uint8_t *d_ = nullptr;
  uint64_t size_ = 0, pos_ = 0;
  bool eof_ = false;
  int fd_ = -1;
  std::vector<uint8_t> stage_, chunk_;
  std::vector<uint64_t> coff_, ooff_, moff_;
  std::vector<uint32_t> crc_;
};

/* FASTA in BGZF (bgzip) members (BgzfMembers), read window by window. */
class BgzfFasta {
 public:
  BgzfFasta() = default;
  BgzfFasta(const BgzfFasta &) = delete;
  /* false if the file cannot be mapped or its first member is not BGZF: the line reader handles it */
  bool open(const std::string &filename) { return mem_.open(filename); }
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
  bool grow(BlockInflater &inf, Buf &b, uint64_t need, std::string &error);
  bool fill(BlockInflater &inf, Buf &b, uint64_t target, std::string &error);

  BgzfMembers mem_;
  std::string error_;
};

/*
 * The one step of the FASTQ window reader that a caller chooses: a window of FASTQ text that grows at its end and is
 * cut into records, with the contract of mm_fastq_append_text / mm_fastq_append_blocks / mm_fastq_cut
 * (include/mashmap_b200.h; record semantics in mm_fastq.h). The program passes DeviceFastqParser; the tests pass
 * HostFastqParser (the host build of mm_fastq.h). Each returns 0, or nonzero with `error` (and *bad_block) set. alloc /
 * release give the reader's staging buffers (pinned ones for the device).
 */
class FastqParser {
 public:
  virtual ~FastqParser() = default;
  virtual int append_text(const uint8_t *text, uint64_t n, std::string &error) = 0;
  virtual int append_blocks(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                            uint64_t n_blocks, int64_t *bad_block, std::string &error) = 0;
  virtual int cut(int last, mm_fastq_records &out, std::string &error) = 0;
  virtual void *alloc(uint64_t bytes);
  virtual void release(void *p);
};

class HostFastqParser : public FastqParser {
 public:
  int append_text(const uint8_t *text, uint64_t n, std::string &error) override;
  int append_blocks(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                    uint64_t n_blocks, int64_t *bad_block, std::string &error) override;
  int cut(int last, mm_fastq_records &out, std::string &error) override;

 private:
  struct Out { std::vector<uint64_t> name_off, nib_off, seq_len; std::string names; std::vector<uint8_t> nibbles; };
  std::vector<uint8_t> win_;
  std::vector<uint64_t> nl_;
  Out out_[2];
  int next_ = 0;
};

class DeviceFastqParser : public FastqParser {
 public:
  /* exits the program (status 1) if the device cannot be used */
  explicit DeviceFastqParser(int device);
  ~DeviceFastqParser() override;
  int append_text(const uint8_t *text, uint64_t n, std::string &error) override;
  int append_blocks(const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off, const uint32_t *crc,
                    uint64_t n_blocks, int64_t *bad_block, std::string &error) override;
  int cut(int last, mm_fastq_records &out, std::string &error) override;
  void *alloc(uint64_t bytes) override;
  void release(void *p) override;

 private:
  mm_fastq *fq_ = nullptr;
};

/*
 * FASTQ read window by window through a FastqParser: a plain file (mapped, staged by the host threads and appended as
 * text) or a BGZF one (BgzfMembers: BGZF runs appended as blocks, zlib members as text). The records are exactly the line
 * reader's (mm_fastq.h).
 */
class FastqReader {
 public:
  FastqReader() = default;
  ~FastqReader();
  FastqReader(const FastqReader &) = delete;
  /* false unless the file is plain or BGZF and its text starts with '@': the line reader handles it */
  bool open(const std::string &filename);
  bool bgzf() const { return bgzf_; }
  /*
   * Appends about window_bytes of text at a time (more while one record does not fit), cuts the window, and hands each
   * cut's records to fn, in order. Window i+1 is appended and cut while fn runs on window i. Stops after an empty line in
   * header position. Returns 0, or -1 on an error (error() says which; a corrupt member: the file and its byte offset).
   */
  int for_each_window(FastqParser &p, uint64_t window_bytes, int threads, const std::function<void(const mm_fastq_records &)> &fn);
  const std::string &error() const { return error_; }

 private:
  bool load(FastqParser &p, uint64_t target, int threads);
  bool at_end() const { return bgzf_ ? mem_.at_end() : pos_ == size_; }

  std::string path_, error_;
  bool bgzf_ = false;
  BgzfMembers mem_;
  const uint8_t *d_ = nullptr; /* plain: the mapped file */
  uint64_t size_ = 0, pos_ = 0;
  int fd_ = -1;
  uint64_t held_ = 0;          /* bytes in the parser's window */
  uint8_t *stage_ = nullptr;    /* plain: pinned staging from the parser, for one for_each_window */
  uint64_t stage_cap_ = 0;
};

/* text bytes per BGZF window for a run of --batchBases b: b, kept within [64 KiB, 256 MiB] */
uint64_t bgzf_window_bytes(uint64_t batch_bases);

/* text bytes per FASTQ window for a run of --batchBases b: 2 b (a FASTQ record's text is about twice its bases: the
 * quality line), kept within [64 KiB, 512 MiB] */
uint64_t fastq_window_bytes(uint64_t batch_bases);

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
