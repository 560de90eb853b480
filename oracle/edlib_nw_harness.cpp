// ORACLE / TEST INFRASTRUCTURE ONLY.
// edlibAlign(query, target, k, EDLIB_MODE_NW, EDLIB_TASK_PATH) of the reference's own header-only edlib (compiled
// unmodified), the call mashmap-b200 --align restates, with edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD). Compiled together
// with edlib_harness.cpp (which pulls in edlib), so this library also exports ref_edlib_align. Built into
// oracle/_ref/libedlib_nw_ref.so only where the reference is readable.
#include "edlib_harness.cpp"

extern "C" {

// Same outputs and status as ref_edlib_align.
__attribute__((visibility("default"))) int ref_edlib_align_nw(const char *q, int Q, const char *t, int T, int k, int *ed,
                                                              int *start, int *end, unsigned char *ops, int *n_ops,
                                                              char *cigar, int cigar_cap)
{
  EdlibAlignResult r = edlibAlign(q, Q, t, T, edlibNewAlignConfig(k, EDLIB_MODE_NW, EDLIB_TASK_PATH, NULL, 0));
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
