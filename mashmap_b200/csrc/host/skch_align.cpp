#include "skch_align.hpp"

#include <chrono>
#include <cstdlib>
#include <iostream>

#include "../../../include/mashmap_b200_align.h"

namespace skch {

namespace {

[[noreturn]] void die(const std::string &msg)
{
  std::cerr << "[mashmap-b200] ERROR: --align: " << msg << std::endl;
  exit(1);
}

/* base i of a nibble-packed sequence (seqio::pack_bases: A 0, C 1, T 2, G 3, | 8 for anything else) */
inline uint8_t nibble(const uint8_t *p, uint64_t i) { return (p[i >> 1] >> ((i & 1) * 4)) & 15; }
const char kBase[4] = {'A', 'C', 'T', 'G'};
inline char base(uint8_t x) { return (x & 8) ? 'N' : kBase[x & 3]; }
inline char complement(uint8_t x) { return (x & 8) ? 'N' : kBase[(x & 3) ^ 2]; }  // A <-> T (0, 2), C <-> G (1, 3)

/* edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD): runs of match / mismatch as M, insertion I, deletion D */
void putCigar(std::string &out, const uint8_t *ops, int n)
{
  static const char ch[4] = {'M', 'I', 'D', 'M'};
  for (int i = 0; i < n;) {
    int j = i + 1;
    while (j < n && ch[ops[j]] == ch[ops[i]]) j++;
    out += std::to_string(j - i);
    out += ch[ops[i]];
    i = j;
  }
}

}  // namespace

MappingAligner::MappingAligner(const Parameters &p, const Sketch &r, int device) : param(p), ref(r)
{
  if (mm_align_ctx_create(device, SCRATCH_BYTES, &ctx) != MM_OK)
    die(std::string("mm_align_ctx_create: ") + mm_align_last_error(nullptr));
}

MappingAligner::~MappingAligner() { mm_align_ctx_destroy(ctx); }

void MappingAligner::align(const Item *items, size_t n, std::vector<std::string> &tags)
{
  const auto t0 = std::chrono::steady_clock::now();
  tags.assign(n, std::string());
  std::vector<char> qb, tb;
  std::vector<mm_align_job> jobs;
  std::vector<size_t> owner;  // item of each job
  std::vector<mm_align_result> res;
  std::vector<uint8_t> ops;
  auto flush = [&]() {
    if (jobs.empty()) return;
    res.resize(jobs.size());
    ops.resize(qb.size() + tb.size());  // NW paths are at most Q + T ops
    uint64_t n_ops = 0;
    if (mm_align_batch(ctx, qb.data(), qb.size(), tb.data(), tb.size(), jobs.data(), jobs.size(), res.data(), ops.data(),
                       ops.size(), &n_ops) != MM_OK)
      die(std::string("mm_align_batch: ") + mm_align_last_error(ctx));
    for (size_t j = 0; j < jobs.size(); j++) {
      const mm_align_result &r = res[j];
      // with k = -1 edlib always has a distance; it has no path only where its Hirschberg split meets a one-column
      // target, which takes a query of more than 3 Mbp (DESIGN.md section 10)
      if (r.ed < 0 || r.alignment_length == 0) { unaligned++; continue; }
      std::string &t = tags[owner[j]];
      t = "\tNM:i:" + std::to_string(r.ed) + "\tcg:Z:";
      putCigar(t, ops.data() + r.ops_offset, r.alignment_length);
      aligned++;
    }
    bases += qb.size() + tb.size();
    qb.clear(); tb.clear(); jobs.clear(); owner.clear();
  };
  for (size_t i = 0; i < n; i++) {
    const MappingResult &m = *items[i].m;
    const int64_t qs = m.queryStartPos, ql = (int64_t)m.queryEndPos - qs;
    const int64_t ts = m.refStartPos, tl = (int64_t)m.refEndPos - ts;
    if (ql > param.align_max_len || tl > param.align_max_len) { tooLong++; continue; }
    if (ql <= 0 || tl <= 0) {  // NW of an empty region: every base of the other one is inserted / deleted
      if (ql <= 0 && tl <= 0) { unaligned++; continue; }
      tags[i] = "\tNM:i:" + std::to_string(ql > 0 ? ql : tl) + "\tcg:Z:" + std::to_string(ql > 0 ? ql : tl) + (ql > 0 ? "I" : "D");
      aligned++;
      continue;
    }
    if (!jobs.empty() && qb.size() + tb.size() + (uint64_t)(ql + tl) > BATCH_BASES) flush();
    jobs.push_back(mm_align_job{qb.size(), tb.size(), (int32_t)ql, (int32_t)tl, -1, MM_ALIGN_NW});
    owner.push_back(i);
    const uint8_t *q = items[i].query;
    if (m.strand == strnd::FWD)
      for (int64_t x = qs; x < qs + ql; x++) qb.push_back(base(nibble(q, (uint64_t)x)));
    else
      for (int64_t x = qs + ql - 1; x >= qs; x--) qb.push_back(complement(nibble(q, (uint64_t)x)));
    const uint8_t *t = ref.refNibbles(m.refSeqId);
    for (int64_t x = ts; x < ts + tl; x++) tb.push_back(base(nibble(t, (uint64_t)x)));
  }
  flush();
  seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

void appendTags(std::string &text, const std::string *tags)
{
  std::string out;
  out.reserve(text.size() + text.size() / 2);
  size_t pos = 0;
  for (size_t i = 0; pos < text.size(); i++) {
    const size_t nl = text.find('\n', pos);
    out.append(text, pos, nl - pos);
    out += tags[i];
    out += '\n';
    pos = nl + 1;
  }
  text.swap(out);
}

}  // namespace skch
