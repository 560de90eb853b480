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

inline char lower(char b) { return (char)(b | 0x20); }  // A C G T N -> a c g t n

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
  const uint32_t flags = (param.align_eqx ? MM_ALIGN_TAG_EQX : 0) | (param.align_cs ? MM_ALIGN_TAG_CS : 0);
  tags.assign(n, std::string());
  std::vector<char> qb, tb;
  std::vector<mm_align_job> jobs;
  std::vector<size_t> owner;  // item of each job
  std::vector<mm_align_tag_result> res;
  auto flush = [&]() {
    if (jobs.empty()) return;
    res.resize(jobs.size());
    // a run of L ops takes at most 2L bytes of cg and 3L of cs, and NW paths are at most Q + T ops
    const uint64_t need = (qb.size() + tb.size()) * (param.align_cs ? 5 : 2);
    if (need > textCap) { text.reset(new char[need]); textCap = need; }
    uint64_t n_text = 0;
    if (mm_align_batch_tags(ctx, qb.data(), qb.size(), tb.data(), tb.size(), jobs.data(), jobs.size(), flags, res.data(),
                            text.get(), textCap, &n_text) != MM_OK)
      die(std::string("mm_align_batch_tags: ") + mm_align_last_error(ctx));
    for (size_t j = 0; j < jobs.size(); j++) {
      const mm_align_tag_result &r = res[j];
      // with k = -1 edlib always has a distance; it has no path only where its Hirschberg split meets a one-column
      // target, which takes a query of more than 3 Mbp (DESIGN.md section 10)
      if (r.ed < 0 || r.alignment_length == 0) { unaligned++; continue; }
      std::string &t = tags[owner[j]];
      t = "\tNM:i:" + std::to_string(r.ed) + "\tcg:Z:";
      t.append(text.get() + r.cg_offset, r.cg_len);
      if (param.align_cs) t.append("\tcs:Z:").append(text.get() + r.cs_offset, r.cs_len);
      aligned++;
    }
    bases += qb.size() + tb.size();
    qb.clear(); tb.clear(); jobs.clear(); owner.clear();
  };
  // the query region, reverse-complemented for a '-' mapping, and the target region
  auto query = [&](const MappingResult &m, const uint8_t *q, auto put) {
    const int64_t qs = m.queryStartPos, qe = m.queryEndPos;
    if (m.strand == strnd::FWD)
      for (int64_t x = qs; x < qe; x++) put(base(nibble(q, (uint64_t)x)));
    else
      for (int64_t x = qe - 1; x >= qs; x--) put(complement(nibble(q, (uint64_t)x)));
  };
  auto target = [&](const MappingResult &m, auto put) {
    const uint8_t *t = ref.refNibbles(m.refSeqId);
    for (int64_t x = m.refStartPos; x < (int64_t)m.refEndPos; x++) put(base(nibble(t, (uint64_t)x)));
  };
  for (size_t i = 0; i < n; i++) {
    const MappingResult &m = *items[i].m;
    const int64_t ql = (int64_t)m.queryEndPos - m.queryStartPos, tl = (int64_t)m.refEndPos - m.refStartPos;
    if (ql > param.align_max_len || tl > param.align_max_len) { tooLong++; continue; }
    if (ql <= 0 || tl <= 0) {  // NW of an empty region: every base of the other one is inserted / deleted
      if (ql <= 0 && tl <= 0) { unaligned++; continue; }
      std::string &t = tags[i];
      t = "\tNM:i:" + std::to_string(ql > 0 ? ql : tl) + "\tcg:Z:" + std::to_string(ql > 0 ? ql : tl) + (ql > 0 ? "I" : "D");
      if (param.align_cs) {
        t += ql > 0 ? "\tcs:Z:+" : "\tcs:Z:-";
        auto put = [&](char b) { t += lower(b); };
        if (ql > 0) query(m, items[i].query, put);
        else target(m, put);
      }
      aligned++;
      continue;
    }
    if (!jobs.empty() && qb.size() + tb.size() + (uint64_t)(ql + tl) > BATCH_BASES) flush();
    jobs.push_back(mm_align_job{qb.size(), tb.size(), (int32_t)ql, (int32_t)tl, -1, MM_ALIGN_NW});
    owner.push_back(i);
    query(m, items[i].query, [&](char b) { qb.push_back(b); });
    target(m, [&](char b) { tb.push_back(b); });
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
