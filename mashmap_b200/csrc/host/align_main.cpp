/*
 * align_main.cpp -- mashmap-b200-align: the reference's mashmap-align (src/align) with the edlib calls on the device.
 *
 * Same options (parseCmdArgs.hpp:27-60, plus --device, --batchBases and --dryRun) and the same output file: for every
 * mapping line that edlib aligns, the line verbatim, " ", editDistance / alignmentLength as an ostream prints a double
 * (%g, six significant digits), " ", the EDLIB_CIGAR_STANDARD CIGAR (computeAlignments.hpp:286-296). Restated from
 * computeAlignments.hpp, quirks included:
 *   - subjects are read whole (:70-103); for each query file the mapping file is re-opened and the output file is
 *     re-opened, i.e. truncated (:118-130), so a --queryList leaves only the last file's alignments;
 *   - mapping lines are matched to queries by walking both in order (:132-177): a query without a line is skipped and a
 *     line out of query order is lost, as in the reference;
 *   - regions take inclusive ends (:234, :240); one base past the end of a sequence is its terminating NUL, a symbol
 *     that matches only itself (strncpy pads the query with NUL, reverseComplement keeps it);
 *   - k = (int)((1 - pi / 100) * queryLen) in float, unbounded for pi == 0 (:256-261).
 * Where the reference fails an assert (fewer than 9 fields, a region longer than its sequence, a duplicate subject) or
 * reads outside a sequence, this program stops before any device work, naming the mapping line. The inputs are walked
 * twice for that: once to check every line, once to align.
 */
#include <charconv>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../../include/mashmap_b200_align.h"
#include "skch_seqio.hpp"

namespace {

struct Params {
  std::vector<std::string> refs, queries;
  std::string mapping, output = "mashmap.out.sam";
  float pi = 0;
  int threads = 1;  // parsed and unused, as in the reference
  int device = 0;
  uint64_t batch_bases = 256ull << 20;
  bool dry_run = false;
};

[[noreturn]] void die(const std::string &msg)
{
  std::cerr << msg << std::endl;
  exit(1);
}

void usage()
{
  std::cout << "-----------------\n"
               "Post process mashmap output to compute alignments for obtaining SAM output (edlib on the GPU).\n"
               "Provide same reference, query files that were used for obtaining mashmap mapping boundaries.\n"
               "-----------------\n"
               "Example usage: \n"
               "$ mashmap-b200-align -s ref.fa -q seq.fq --mappingFile mashmap.out --pi 80 [OPTIONS]\n\n"
               "  -s, --subject FILE        an input reference file (fasta/fastq)[.gz]\n"
               "  --sl, --subjectList FILE  a file containing list of reference files, one per line\n"
               "  -q, --query FILE          an input query file (fasta/fastq)[.gz]\n"
               "  --ql, --queryList FILE    a file containing list of query files, one per line\n"
               "  --mappingFile FILE        mashmap file containing mapping information (required)\n"
               "  --pi, --perc_identity X   edlib threshold for alignment identity [0-100] (required)\n"
               "  -t, --threads N           accepted for compatibility; the alignments run on the GPU\n"
               "  -o, --output FILE         output file name [default : mashmap.out.sam]\n"
               "  --device N                CUDA device [default : 0]\n"
               "  --batchBases N            query + target bases aligned per device batch [default : 268435456]\n"
               "  --dryRun                  check the inputs and list the edlib calls, without a device\n"
               "  -h, --help                print this help page\n";
}

void parse_file_list(const std::string &list, std::vector<std::string> &out)
{  // skch::parseFileList (map/include/parseCmdArgs.hpp)
  std::ifstream in(list);
  if (!in) die("ERROR, skch::parseFileList, Could not open " + list);
  std::string line;
  while (std::getline(in, line))
    if (!line.empty()) out.push_back(line);
}

template <class T>
T to(const std::string &s)
{  // parseandSave reads every value through a stringstream (parseCmdArgs.hpp:107-182)
  std::stringstream str;
  str << s;
  T v{};
  str >> v;
  return v;
}

Params parse_args(int argc, char **argv)
{
  static const std::map<std::string, std::pair<std::string, bool>> names = {
      // spelling -> (option, takes a value)
      {"-s", {"subject", true}},       {"--subject", {"subject", true}},     {"--sl", {"subjectList", true}},
      {"--subjectList", {"subjectList", true}}, {"-q", {"query", true}},     {"--query", {"query", true}},
      {"--ql", {"queryList", true}},   {"--queryList", {"queryList", true}}, {"--mappingFile", {"mappingFile", true}},
      {"--pi", {"perc_identity", true}}, {"--perc_identity", {"perc_identity", true}}, {"-t", {"threads", true}},
      {"--threads", {"threads", true}}, {"-o", {"output", true}},           {"--output", {"output", true}},
      {"--device", {"device", true}},  {"--batchBases", {"batchBases", true}}, {"--dryRun", {"dryRun", false}},
      {"-h", {"help", false}},         {"--help", {"help", false}}};
  std::map<std::string, std::string> opt;
  for (int i = 1; i < argc; i++) {
    std::string a = argv[i], val;
    bool has_val = false;
    const size_t eq = a.find('=');
    if (a.rfind("--", 0) == 0 && eq != std::string::npos) { val = a.substr(eq + 1); a = a.substr(0, eq); has_val = true; }
    auto it = names.find(a);
    if (it == names.end()) die("Unknown option " + a);
    if (it->second.second && !has_val) {
      if (i + 1 >= argc) die("Option " + a + " requires a value");
      val = argv[++i];
    }
    opt[it->second.first] = val;
  }
  if (opt.count("help")) { usage(); exit(0); }
  if (!opt.count("mappingFile")) die("Required option missing: mappingFile");
  if (!opt.count("perc_identity")) die("Required option missing: perc_identity");
  if (!opt.count("subject") && !opt.count("subjectList"))
    die("ERROR, align::parseandSave, Provide reference file(s)\n"
        "        This input should be same as used for generating mashmap mapping output");
  if (!opt.count("query") && !opt.count("queryList"))
    die("ERROR, align::parseandSave, Provide query file(s)\n"
        "        This input should be same as used for generating mashmap mapping output");
  Params p;
  if (opt.count("subject")) p.refs.push_back(to<std::string>(opt["subject"]));
  else parse_file_list(to<std::string>(opt["subjectList"]), p.refs);
  if (opt.count("query")) p.queries.push_back(to<std::string>(opt["query"]));
  else parse_file_list(to<std::string>(opt["queryList"]), p.queries);
  p.mapping = to<std::string>(opt["mappingFile"]);
  p.pi = to<float>(opt["perc_identity"]);
  if (opt.count("threads")) p.threads = to<int>(opt["threads"]);
  if (opt.count("output")) p.output = to<std::string>(opt["output"]);
  if (opt.count("device")) p.device = to<int>(opt["device"]);
  if (opt.count("batchBases")) {
    const long long b = to<long long>(opt["batchBases"]);
    if (b < 1) die("ERROR, --batchBases must be a positive number of bases");
    p.batch_bases = (uint64_t)b;
  }
  p.dry_run = opt.count("dryRun") != 0;

  std::cout << ">>>>>>>>>>>>>>>>>>" << std::endl;
  auto list = [](const std::vector<std::string> &v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); i++) s += (i ? ", " : "") + v[i];
    return s + "]";
  };
  std::cout << "Reference = " << list(p.refs) << std::endl;
  std::cout << "Query = " << list(p.queries) << std::endl;
  std::cout << "Mapping file = " << p.mapping << std::endl;
  std::cout << "Edlib identity cut-off = " << p.pi << "%" << std::endl;
  std::cout << "Alignment output file = " << p.output << std::endl;
  std::cout << ">>>>>>>>>>>>>>>>>>" << std::endl;

  if (!std::ifstream(p.mapping)) die("ERROR, skch::validateInputFile, Could not open " + p.mapping);
  for (const auto &f : p.queries)
    if (!std::ifstream(f)) die("ERROR, skch::validateInputFiles, Could not open " + f);
  for (const auto &f : p.refs)
    if (!std::ifstream(f)) die("ERROR, skch::validateInputFiles, Could not open " + f);
  return p;
}

/* CommonFunc::makeUpperCaseAndValidDNA (commonFunc.hpp:97-107): lower case to upper, anything but ACGT to N */
void normalise(std::string &s)
{
  for (char &c : s) {
    if (c > 96 && c < 123) c -= 32;
    if (c != 'A' && c != 'C' && c != 'G' && c != 'T') c = 'N';
  }
}

struct Record {  // MappingBoundaryRow (align_types.hpp), parsed as parseMashmapRow does (computeAlignments.hpp:191-214)
  std::string qId, refId;
  int qStart = 0, qEnd = 0, rStart = 0, rEnd = 0;
  bool fwd = true;
};

struct Job {
  std::string line;
  int64_t q_off, t_off;
  int q_len, t_len, k;
};

class Aligner {
 public:
  explicit Aligner(const Params &p) : p_(p) {}

  void read_subjects()
  {
    for (const auto &f : p_.refs) {
      const bool ok = skch::seqio::for_each_seq_in_file(f, {}, "", [&](const std::string &name, const std::string &seq) {
        if (refs_.count(name)) die("ERROR, mashmap-b200-align: subject sequence " + name + " appears twice (the reference aligner asserts)");
        std::string s = seq;
        normalise(s);
        refs_.emplace(name, std::move(s));
      });
      if (!ok) exit(1);
    }
  }

  /* pass 0 checks every line without a device; pass 1 aligns */
  void run(int pass)
  {
    pass_ = pass;
    for (const auto &qf : p_.queries) {
      if (pass == 1 && !p_.dry_run) {
        out_.close();
        out_.open(p_.output, std::ios::out | std::ios::trunc);  // re-opened for every query file (:130)
        if (!out_) die("ERROR, mashmap-b200-align: cannot write " + p_.output);
      }
      std::ifstream maps(p_.mapping);
      std::string line;
      long line_no = 0;
      bool done = false;
      Record rec;
      const bool ok = skch::seqio::for_each_seq_in_file(qf, {}, "", [&](const std::string &name, const std::string &seq0) {
        if (done) return;
        if (maps.eof()) { done = true; return; }  // :140-141
        std::string seq = seq0;
        normalise(seq);
        if (line.empty()) { std::getline(maps, line); line_no++; }  // :144-147
        parse(line, line_no, rec);
        if (rec.qId != name) return;  // :152-156
        add(rec, line, line_no, seq);
        while (std::getline(maps, line)) {  // :163-176
          line_no++;
          parse(line, line_no, rec);
          if (rec.qId != name) break;
          add(rec, line, line_no, seq);
        }
      });
      if (!ok) exit(1);
      if (pass == 1) flush();
    }
    if (pass == 1 && !p_.dry_run) out_.close();
  }

  void open_device()
  {
    const int rc = mm_align_ctx_create(p_.device, 0, &ctx_);
    if (rc != MM_OK) die(std::string("ERROR, mashmap-b200-align: ") + mm_align_last_error(nullptr));
  }
  ~Aligner()
  {
    if (ctx_) mm_align_ctx_destroy(ctx_);
  }
  double device_ms() const { return device_ms_; }
  uint64_t aligned() const { return aligned_; }

 private:
  void parse(const std::string &line, long line_no, Record &r)
  {
    std::stringstream ss(line);
    std::string w;
    std::vector<std::string> tok;
    while (ss >> w) tok.push_back(w);
    if (tok.size() < 9)
      die("ERROR, mashmap-b200-align: mapping line " + std::to_string(line_no) + " has fewer than 9 fields "
          "(the reference aligner asserts): \"" + line + "\"");
    try {
      r.qId = tok[0];
      r.qStart = std::stoi(tok[2]);
      r.qEnd = std::stoi(tok[3]);
      r.fwd = tok[4] == "+";
      r.refId = tok[5];
      r.rStart = std::stoi(tok[7]);
      r.rEnd = std::stoi(tok[8]);
    } catch (const std::exception &) {
      die("ERROR, mashmap-b200-align: mapping line " + std::to_string(line_no) + " has a non-numeric coordinate: \"" + line + "\"");
    }
  }

  /* the region [start, start + len) of s, where index s.size() is the string's NUL; false if the reference would fail its
   * assert (len > size) or read outside the string */
  static bool region_ok(const std::string &s, long long start, long long len)
  {
    return len >= 1 && len <= (long long)s.size() && start >= 0 && start + len <= (long long)s.size() + 1;
  }

  void add(const Record &r, const std::string &line, long line_no, const std::string &qseq)
  {
    auto fail = [&](const std::string &why) {
      die("ERROR, mashmap-b200-align: mapping line " + std::to_string(line_no) + ": " + why + ": \"" + line + "\"");
    };
    auto it = refs_.find(r.refId);
    if (it == refs_.end()) fail("subject sequence " + r.refId + " is not in the subject files");
    const std::string &ref = it->second;
    const long long refLen = (long long)r.rEnd - r.rStart + 1, queryLen = (long long)r.qEnd - r.qStart + 1;
    if (!region_ok(ref, r.rStart, refLen))
      fail("subject region " + std::to_string(r.rStart) + ".." + std::to_string(r.rEnd) + " does not fit " + r.refId +
           " (length " + std::to_string(ref.size()) + ")");
    if (!region_ok(qseq, r.qStart, queryLen))
      fail("query region " + std::to_string(r.qStart) + ".." + std::to_string(r.qEnd) + " does not fit " + r.qId +
           " (length " + std::to_string(qseq.size()) + ")");
    int k = -1;
    if (p_.pi != 0) {
      const float f = (1 - p_.pi / 100) * (float)queryLen;  // float arithmetic, truncated (:261)
      k = (int)f;
    }
    if (pass_ == 0) return;
    if (p_.dry_run) {
      std::cout << "edlib " << line_no << ' ' << r.qId << ' ' << r.qStart << ' ' << queryLen << ' ' << (r.fwd ? '+' : '-')
                << ' ' << r.refId << ' ' << r.rStart << ' ' << refLen << ' ' << k << '\n';
      return;
    }
    Job j;
    j.line = line;
    j.q_off = (int64_t)qbuf_.size();
    j.t_off = (int64_t)tbuf_.size();
    j.q_len = (int)queryLen;
    j.t_len = (int)refLen;
    j.k = k;
    auto at = [](const std::string &s, long long i) -> char { return i < (long long)s.size() ? s[i] : '\0'; };
    for (long long i = 0; i < refLen; i++) tbuf_.push_back(at(ref, r.rStart + i));
    if (r.fwd) {
      for (long long i = 0; i < queryLen; i++) qbuf_.push_back(at(qseq, r.qStart + i));
    } else {  // CommonFunc::reverseComplement: ACGT complemented, N and NUL kept
      for (long long i = queryLen - 1; i >= 0; i--) {
        const char c = at(qseq, r.qStart + i);
        qbuf_.push_back(c == 'A' ? 'T' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == 'T' ? 'A' : c);
      }
    }
    jobs_.push_back(std::move(j));
    if (qbuf_.size() + tbuf_.size() >= p_.batch_bases) flush();
  }

  void flush()
  {
    if (jobs_.empty()) return;
    std::vector<mm_align_job> tab(jobs_.size());
    uint64_t cap = 0;
    for (size_t i = 0; i < jobs_.size(); i++) {
      tab[i] = mm_align_job{(uint64_t)jobs_[i].q_off, (uint64_t)jobs_[i].t_off, jobs_[i].q_len, jobs_[i].t_len, jobs_[i].k, 0};
      cap += (uint64_t)jobs_[i].q_len + jobs_[i].t_len;
    }
    std::vector<mm_align_result> res(jobs_.size());
    std::vector<uint8_t> ops(cap);
    uint64_t n_ops = 0;
    const int rc = mm_align_batch(ctx_, qbuf_.data(), qbuf_.size(), tbuf_.data(), tbuf_.size(), tab.data(), tab.size(),
                                  res.data(), ops.data(), cap, &n_ops);
    if (rc != MM_OK) die(std::string("ERROR, mashmap-b200-align: device alignment failed: ") + mm_align_last_error(ctx_));
    float ms[8];
    mm_align_last_stage_ms(ctx_, ms);
    device_ms_ += ms[6];
    std::string text;
    static const char code[4] = {'M', 'I', 'D', 'M'};
    for (size_t i = 0; i < jobs_.size(); i++) {
      const mm_align_result &r = res[i];
      if (r.ed < 0 || r.alignment_length == 0) continue;  // :286
      aligned_++;
      text += jobs_[i].line;
      text += ' ';
      char buf[64];
      auto e = std::to_chars(buf, buf + sizeof buf, r.ed * 1.0 / r.alignment_length, std::chars_format::general, 6);
      text.append(buf, e.ptr);  // what `os << double` prints (%g, precision 6), as skch_tail's formatter
      text += ' ';
      const uint8_t *o = ops.data() + r.ops_offset;
      for (int a = 0; a < r.alignment_length;) {  // edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD), edlib.hxx:262-311
        const char c = code[o[a]];
        int b = a + 1;
        while (b < r.alignment_length && code[o[b]] == c) b++;
        auto e2 = std::to_chars(buf, buf + sizeof buf, b - a);
        text.append(buf, e2.ptr);
        text += c;
        a = b;
      }
      text += '\n';
    }
    out_ << text;
    jobs_.clear();
    qbuf_.clear();
    tbuf_.clear();
  }

  const Params &p_;
  int pass_ = 0;
  std::unordered_map<std::string, std::string> refs_;
  std::ofstream out_;
  mm_align_ctx *ctx_ = nullptr;
  std::vector<Job> jobs_;
  std::string qbuf_, tbuf_;
  double device_ms_ = 0;
  uint64_t aligned_ = 0;
};

}  // namespace

int main(int argc, char **argv)
{
  std::ios::sync_with_stdio(false);
  const Params p = parse_args(argc, argv);
  const auto t0 = std::chrono::steady_clock::now();
  Aligner a(p);
  a.read_subjects();
  a.run(0);  // every mapping line checked before any device work
  if (!p.dry_run) a.open_device();
  const auto t1 = std::chrono::steady_clock::now();
  std::cout << "INFO, align::main, Time spent read the reference sequences: "
            << std::chrono::duration<double>(t1 - t0).count() << " sec" << std::endl;
  a.run(1);
  const auto t2 = std::chrono::steady_clock::now();
  std::cout << "INFO, align::main, Time spent computing the aligment: " << std::chrono::duration<double>(t2 - t0).count()
            << " sec (device " << a.device_ms() / 1000 << " sec, " << a.aligned() << " alignments)" << std::endl;
  if (!p.dry_run) std::cout << "INFO, align::main, alignment results saved in: " << p.output << std::endl;
  return 0;
}
