// ORACLE / TEST INFRASTRUCTURE ONLY.
// A plain full-matrix CPU restatement of edlibAlign(query, target, k, EDLIB_MODE_NW, EDLIB_TASK_PATH), the call
// mashmap-b200 --align makes on every mapping (DESIGN.md section 10), written from the rules, not from edlib's code.
// Rule 3 (the path) is align_oracle.cpp's, compiled in from that file so that both restatements share it; this library
// therefore also exports ora_align. tests/test_align_nw_cpu.py checks ora_align_nw against the unmodified edlib
// (oracle/_ref/libedlib_nw_ref.so) on random pairs; the GPU tests check the device's NW mode against either.
#include "align_oracle.cpp"

extern "C" {

// Same outputs as ora_align. Rule 1': ed = D[Q-1][T-1] of the full NW matrix, -1 when k >= 0 and ed > k; start 0,
// end T-1. Rule 3 over the whole target with score ed.
__attribute__((visibility("default"))) int ora_align_nw(const unsigned char *q, int Q, const unsigned char *t, int T,
                                                        int k, int *ed, int *start, int *end, unsigned char *ops,
                                                        int *n_ops)
{
  *ed = -1; *start = *end = -1; *n_ops = 0;
  const int best = nw_last_column(Q, T, [&](int i) { return q[i]; }, [&](int j) { return t[j]; })[Q - 1];
  if (k >= 0 && best > k) return 0;
  *ed = best; *start = 0; *end = T - 1;
  std::vector<unsigned char> out;
  if (!obtain(q, Q, t, T, best, out)) return 0;
  std::copy(out.begin(), out.end(), ops);
  *n_ops = (int)out.size();
  return 0;
}

}  // extern "C"
