// ORACLE / TEST INFRASTRUCTURE ONLY.
// Exposes the reference's own header-only edlib (src/common/edlib.hxx, compiled unmodified) as a C function that runs
// edlibAlign(query, target, k, EDLIB_MODE_HW, EDLIB_TASK_PATH) -- the call computeAlignments.hpp:268 makes -- and
// edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD). Built into oracle/_ref/libedlib_ref.so only where the reference is readable.
#include <cstdlib>
#include <cstring>
#include <limits>  // edlib.hxx uses std::numeric_limits and relies on its includer for the header

#include "edlib.h"  // pulls in edlib.hxx, the implementation, at its end

extern "C" {

// Returns edlib's status. ops needs alignmentLength bytes (<= Q + T); cigar (may be NULL) cigar_cap bytes.
__attribute__((visibility("default"))) int ref_edlib_align(const char *q, int Q, const char *t, int T, int k, int *ed,
                                                           int *start, int *end, unsigned char *ops, int *n_ops,
                                                           char *cigar, int cigar_cap)
{
  EdlibAlignResult r = edlibAlign(q, Q, t, T, edlibNewAlignConfig(k, EDLIB_MODE_HW, EDLIB_TASK_PATH, NULL, 0));
  *ed = r.editDistance;
  *start = r.startLocations ? r.startLocations[0] : -1;
  *end = r.endLocations ? r.endLocations[0] : -1;
  *n_ops = r.alignmentLength;
  if (r.alignment && r.alignmentLength > 0) memcpy(ops, r.alignment, r.alignmentLength);
  if (cigar && cigar_cap > 0) {
    cigar[0] = 0;
    if (r.alignment && r.alignmentLength > 0) {
      char *c = edlibAlignmentToCigar(r.alignment, r.alignmentLength, EDLIB_CIGAR_STANDARD);
      if (c) { strncpy(cigar, c, cigar_cap - 1); cigar[cigar_cap - 1] = 0; free(c); }
    }
  }
  const int st = r.status;
  edlibFreeAlignResult(r);
  return st;
}

}  // extern "C"
