// ORACLE / TEST INFRASTRUCTURE ONLY.
// The static-band restatement of edlibAlign(query, target, k, EDLIB_MODE_NW, EDLIB_TASK_PATH) (DESIGN.md section 10):
// the full-matrix rules of align_nw_oracle.cpp, except that every NW sweep whose decision the device takes from a banded
// sweep sees only the cells with |d| + |d - D| <= k (d = i - j, D = Q - T) and +infinity elsewhere:
//   * the distance: k >= 0 and |D| > k gives -1; otherwise one banded pass with k, accepted when <= k. k < 0: banded
//     passes with k = 64, 128, ... until one is accepted.
//   * every Hirschberg node: both half-columns banded with k = the node's score in the node's own (Q, T); rows
//     outside the band take part in the split test as +infinity.
// Leaves are the full-matrix traceback. Applied to every size (the device bands only long sub-problems), so that small
// random pairs exercise the claim. tests/test_align_band_cpu.py checks ora_align_band_nw against ora_align_nw.
#include "align_oracle.cpp"

namespace {

constexpr int INF = 1 << 29;

struct BandRule {
  long long dmin, dmax;
  BandRule(int Q, int T, int k)
  {
    const long long D = (long long)Q - T, ad = D < 0 ? -D : D;
    const long long w = k > ad ? (k - ad) / 2 : 0;
    dmin = std::min(0LL, D) - w;
    dmax = std::max(0LL, D) + w;
  }
  bool in(int i, int j) const { return i - j >= dmin && i - j <= dmax; }
};

// nw_last_column with the cells outside the band (in the view's coordinates) at +infinity; the boundary row and column
// keep their exact values
template <class QF, class TF>
Col band_last_column(int Q, int n, QF q, TF t, const BandRule &band)
{
  Col col(Q);
  for (int i = 0; i < Q; i++) col[i] = i + 1;
  for (int j = 0; j < n; j++) {
    int diag = j, up = j + 1;
    const unsigned char c = t(j);
    for (int i = 0; i < Q; i++) {
      const int left = col[i];
      const int v = band.in(i, j) ? std::min({diag + (q(i) == c ? 0 : 1), up + 1, left + 1, INF}) : INF;
      diag = left;
      col[i] = v;
      up = v;
    }
  }
  return col;
}

bool obtain_band(const unsigned char *q, int Q, const unsigned char *t, int T, int best, std::vector<unsigned char> &out)
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
  if (lw == 0) return false;
  const BandRule band(Q, T, best);
  const Col left = band_last_column(Q, lw, [&](int i) { return q[i]; }, [&](int j) { return t[j]; }, band);
  const Col rrev = band_last_column(Q, rw, [&](int i) { return q[Q - 1 - i]; }, [&](int j) { return t[T - 1 - j]; }, band);
  auto right = [&](int i) { return rrev[Q - 1 - i]; };
  int split = INT_MIN, ls = 0, rs = 0;
  for (int i = 0; i + 1 < Q; i++)
    if (left[i] + right(i + 1) == best) { split = i; ls = left[i]; rs = right(i + 1); break; }
  if (split == INT_MIN && lw + right(0) == best) { split = -1; ls = lw; rs = right(0); }
  if (split == INT_MIN && left[Q - 1] + rw == best) { split = Q - 1; ls = left[Q - 1]; rs = rw; }
  if (split == INT_MIN) return false;
  const int ulh = split + 1;
  if (!obtain_band(q, ulh, t, lw, ls, out)) return false;
  return obtain_band(q + ulh, Q - ulh, t + lw, rw, rs, out);
}

int band_distance(const unsigned char *q, int Q, const unsigned char *t, int T, int k)
{
  return band_last_column(Q, T, [&](int i) { return q[i]; }, [&](int j) { return t[j]; }, BandRule(Q, T, k))[Q - 1];
}

}  // namespace

extern "C" {

// Same outputs as ora_align_nw.
__attribute__((visibility("default"))) int ora_align_band_nw(const unsigned char *q, int Q, const unsigned char *t,
                                                             int T, int k, int *ed, int *start, int *end,
                                                             unsigned char *ops, int *n_ops)
{
  *ed = -1; *start = *end = -1; *n_ops = 0;
  int best;
  if (k >= 0) {
    if (std::abs(Q - T) > k) return 0;
    best = band_distance(q, Q, t, T, k);
    if (best > k) return 0;
  } else {
    for (long long kk = 64;; kk *= 2) {
      best = band_distance(q, Q, t, T, (int)std::min<long long>(kk, INT_MAX));
      if (best <= kk) break;
    }
  }
  *ed = best; *start = 0; *end = T - 1;
  std::vector<unsigned char> out;
  if (!obtain_band(q, Q, t, T, best, out)) return 0;
  std::copy(out.begin(), out.end(), ops);
  *n_ops = (int)out.size();
  return 0;
}

}  // extern "C"
