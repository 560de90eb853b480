// ORACLE / TEST INFRASTRUCTURE ONLY.
// A plain full-matrix CPU restatement of the three decisions edlibAlign(query, target, k, EDLIB_MODE_HW,
// EDLIB_TASK_PATH) makes (DESIGN.md section 10), written from the rules, not from edlib's code. Nothing here is band
// limited: every cell of every matrix is exact. tests/test_align_cpu.py checks it against the unmodified edlib
// (oracle/_ref/libedlib_ref.so) on random pairs; the GPU tests check the device path against either.
//
// Edit ops use edlib's codes: 0 match, 1 insertion (query base not in target), 2 deletion, 3 mismatch.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

namespace {

typedef std::vector<int> Col;

// NW last column: D[i][n-1] for i in 0..Q-1 of query q vs target t[0..n), D[-1][j] = j + 1, D[i][-1] = i + 1.
// q / t are read through index maps so reversed views need no copies.
template <class QF, class TF>
Col nw_last_column(int Q, int n, QF q, TF t)
{
  Col col(Q);
  for (int i = 0; i < Q; i++) col[i] = i + 1;
  for (int j = 0; j < n; j++) {
    int diag = j;          // D[-1][j-1]
    int up = j + 1;        // D[-1][j]
    const unsigned char c = t(j);
    for (int i = 0; i < Q; i++) {
      const int left = col[i];
      const int v = std::min({diag + (q(i) == c ? 0 : 1), up + 1, left + 1});
      diag = left;
      col[i] = v;
      up = v;
    }
  }
  return col;
}

// Rule 3, leaf: the traceback over the full NW matrix with edlib's move preference (up, then left, then diagonal).
void traceback(const unsigned char *q, int Q, const unsigned char *t, int T, std::vector<unsigned char> &out)
{
  std::vector<int> D((size_t)(Q + 1) * (T + 1));
  auto at = [&](int i, int j) -> int & { return D[(size_t)(i + 1) * (T + 1) + (j + 1)]; };
  for (int j = -1; j < T; j++) at(-1, j) = j + 1;
  for (int i = 0; i < Q; i++) {
    at(i, -1) = i + 1;
    for (int j = 0; j < T; j++)
      at(i, j) = std::min({at(i - 1, j - 1) + (q[i] == t[j] ? 0 : 1), at(i - 1, j) + 1, at(i, j - 1) + 1});
  }
  std::vector<unsigned char> ops;
  int i = Q - 1, j = T - 1;
  while (true) {
    if (i == -1) { for (int x = 0; x <= j; x++) ops.push_back(2); break; }
    if (j == -1) { for (int x = 0; x <= i; x++) ops.push_back(1); break; }
    const int cur = at(i, j);
    if (at(i - 1, j) + 1 == cur) { ops.push_back(1); i--; }
    else if (at(i, j - 1) + 1 == cur) { ops.push_back(2); j--; }
    else { ops.push_back(at(i - 1, j - 1) == cur ? 0 : 3); i--; j--; }
  }
  out.insert(out.end(), ops.rbegin(), ops.rend());
}

// Rule 3: traceback when edlib's stored-block estimate is under 1 MiB, Hirschberg otherwise. false = no split row
// (edlib then returns no alignment).
bool obtain(const unsigned char *q, int Q, const unsigned char *t, int T, int best, std::vector<unsigned char> &out)
{
  if (Q == 0 || T == 0) {
    for (int x = 0; x < Q + T; x++) out.push_back(Q == 0 ? 2 : 1);
    return true;
  }
  const long long nb = (Q + 63) / 64;
  if ((2 * 8 + 4) * nb * T + 2 * 4 * (long long)T < 1024 * 1024) {
    traceback(q, Q, t, T, out);
    return true;
  }
  const int lw = T / 2, rw = T - lw;
  const Col left = nw_last_column(Q, lw, [&](int i) { return q[i]; }, [&](int j) { return t[j]; });
  const Col rrev = nw_last_column(Q, rw, [&](int i) { return q[Q - 1 - i]; }, [&](int j) { return t[T - 1 - j]; });
  auto right = [&](int i) { return rrev[Q - 1 - i]; };  // NW(q[i..Q), t[lw..T))
  int split = INT_MIN, ls = 0, rs = 0;
  for (int i = 0; i + 1 < Q; i++)
    if (left[i] + right(i + 1) == best) { split = i; ls = left[i]; rs = right(i + 1); break; }
  if (split == INT_MIN && lw + right(0) == best) { split = -1; ls = lw; rs = right(0); }
  if (split == INT_MIN && left[Q - 1] + rw == best) { split = Q - 1; ls = left[Q - 1]; rs = rw; }
  if (split == INT_MIN) return false;
  const int ulh = split + 1;
  if (!obtain(q, ulh, t, lw, ls, out)) return false;
  return obtain(q + ulh, Q - ulh, t + lw, rw, rs, out);
}

}  // namespace

extern "C" {

// Returns 0. ed = -1 when no alignment is within k (then nothing else is set). ops needs Q + T bytes.
__attribute__((visibility("default"))) int ora_align(const unsigned char *q, int Q, const unsigned char *t, int T,
                                                     int k, int *ed, int *start, int *end, unsigned char *ops,
                                                     int *n_ops)
{
  *ed = -1; *start = *end = -1; *n_ops = 0;
  // Rule 1: HW last row (free start on the target), smallest column with the minimum. When Q is not a multiple of 64,
  // column -1 (empty target prefix, score Q) takes part and wins ties.
  int best = (Q % 64) ? Q : INT_MAX, bestpos = -1;
  {
    std::vector<int> col(Q);
    for (int i = 0; i < Q; i++) col[i] = i + 1;
    for (int j = 0; j < T; j++) {
      int diag = 0, up = 0;
      for (int i = 0; i < Q; i++) {
        const int l = col[i];
        const int v = std::min({diag + (q[i] == t[j] ? 0 : 1), up + 1, l + 1});
        diag = l; col[i] = v; up = v;
      }
      if (col[Q - 1] < best) { best = col[Q - 1]; bestpos = j; }
    }
  }
  const int kk = k < 0 ? INT_MAX : std::min(k, Q);
  if (best > kk) return 0;
  *ed = best; *end = bestpos;
  // Rule 2: start = end - (largest position of the minimum in the SHW pass of the reversed query over the reversed
  // target prefix [0, end]).
  if (bestpos < 0) {
    *start = 0;
  } else {
    const int n = bestpos + 1;
    std::vector<int> col(Q);
    for (int i = 0; i < Q; i++) col[i] = i + 1;
    int m = INT_MAX, mpos = -1;
    for (int j = 0; j < n; j++) {
      const unsigned char c = t[bestpos - j];
      int diag = j, up = j + 1;
      for (int i = 0; i < Q; i++) {
        const int l = col[i];
        const int v = std::min({diag + (q[Q - 1 - i] == c ? 0 : 1), up + 1, l + 1});
        diag = l; col[i] = v; up = v;
      }
      if (col[Q - 1] <= m) { m = col[Q - 1]; mpos = j; }
    }
    *start = bestpos - mpos;
  }
  std::vector<unsigned char> out;
  if (!obtain(q, Q, t + *start, *end - *start + 1, best, out)) return 0;
  std::copy(out.begin(), out.end(), ops);
  *n_ops = (int)out.size();
  return 0;
}

}  // extern "C"
