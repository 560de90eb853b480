/*
 * skch_align.hpp -- mashmap-b200 --align: base-level alignment of the mappings the run prints.
 *
 * Every printed mapping's exact PAF region is aligned end to end with edlib's global mode (EDLIB_MODE_NW,
 * EDLIB_TASK_PATH, k = -1) on the device (mm_align_batch_tags, MM_ALIGN_NW jobs, include/mashmap_b200_align.h):
 *   query  = [qStart, qEnd) of the normalised query (ACGT, everything else N), reverse-complemented for a '-' mapping
 *            (CommonFunc::reverseComplement: ACGT complemented, N kept);
 *   target = [tStart, tEnd) of the normalised reference contig.
 * The line gets "\tNM:i:<edit distance>\tcg:Z:<CIGAR>" (edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD): M / I / D; with
 * --eqx EDLIB_CIGAR_EXTENDED: = / X / I / D), so the CIGAR consumes exactly the bases columns 3-4 and 8-9 describe. With
 * --cs the line also gets "\tcs:Z:<minimap2's short difference string>" of the same path, in the same orientation. The
 * tag text is written on the device (mm_align_batch_tags); only the text comes back. A mapping whose query or target
 * region is longer than --alignMaxLen is printed without the tags. A tag depends on its mapping alone, never on the batch
 * it was aligned in.
 */
#ifndef SKCH_ALIGN_HPP
#define SKCH_ALIGN_HPP

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "skch_index.hpp"
#include "skch_types.hpp"

struct mm_align_ctx;

namespace skch {

class MappingAligner {
 public:
  /* Device memory bound of one aligner (one per device): mm_align_batch_tags calls of at most BATCH_BASES query + target
   * bases (inputs and edit-op buffer: 2 x 256 MiB), a kernel scratch budget of SCRATCH_BYTES (work beyond it runs in
   * waves) and the tag formatting pass's arrays (about a quarter of it), about 3 GiB beside the mapping contexts of the
   * same device. */
  static constexpr uint64_t BATCH_BASES = 256ull << 20;
  static constexpr uint64_t SCRATCH_BYTES = 2ull << 30;

  MappingAligner(const Parameters &p, const Sketch &ref, int device);
  ~MappingAligner();
  MappingAligner(const MappingAligner &) = delete;

  struct Item {
    const MappingResult *m;
    const uint8_t *query;  // the nibbles (seqio::pack_bases) of m's whole query, base 0 in the low nibble of byte 0
  };
  /* tags[i] = the tags of items[i] ("" when it is not aligned) */
  void align(const Item *items, size_t n, std::vector<std::string> &tags);

  // totals over the run: mappings with tags, mappings over --alignMaxLen, mappings edlib gives no path for (both regions
  // empty), query + target bases sent to the device, seconds spent in align()
  uint64_t aligned = 0, tooLong = 0, unaligned = 0, bases = 0;
  double seconds = 0;

 private:
  const Parameters &param;
  const Sketch &ref;
  mm_align_ctx *ctx = nullptr;
  std::unique_ptr<char[]> text;  // tag text of one batch, left uninitialised: only what the device writes is touched
  uint64_t textCap = 0;
};

/* text holds one '\n'-terminated line per mapping; appends tags[i] to the end of line i */
void appendTags(std::string &text, const std::string *tags);

}  // namespace skch
#endif
