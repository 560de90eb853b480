/* ORACLE / TEST INFRASTRUCTURE ONLY -- never linked into the product.
 *
 * Stand-in for the three GNU Scientific Library functions the reference calls
 * (GSL is a system dependency of marbl/MashMap, un-vendored and un-pinned:
 * INSTALL.txt:7, CMakeLists.txt:92-93):
 *   gsl_cdf_binomial_Q          map_stats.hpp:98,213
 *   gsl_ran_hypergeometric_pdf  computeMap.hpp:194
 *   gsl_cdf_hypergeometric_P    computeMap.hpp:213
 * Their values only feed threshold comparisons that yield integers (SURVEY 8(c)).
 * "parity unpinned" at the GSL boundary: the reference ships no test that pins
 * these values; tests/test_stats.py checks that the integer decisions of this
 * stand-in (log-gamma start term + one-sided term recurrence) equal those of the
 * product's independent implementation.
 */
#ifndef MM_ORACLE_GSL_CDF_H
#define MM_ORACLE_GSL_CDF_H

#include <math.h>

#ifdef __cplusplus
extern "C" {
#endif

static inline double mm_shim_lnchoose(unsigned int n, unsigned int m)
{
  if (m > n) return -INFINITY;
  return lgamma((double)n + 1.0) - lgamma((double)m + 1.0) - lgamma((double)(n - m) + 1.0);
}

/* log of the binomial pmf at i */
static inline double mm_shim_binom_logpmf(unsigned int i, double p, unsigned int n)
{
  return mm_shim_lnchoose(n, i) + (double)i * log(p) + (double)(n - i) * log1p(-p);
}

/* P(X > k), X ~ Binomial(n, p) */
static inline double gsl_cdf_binomial_Q(const unsigned int k, const double p, const unsigned int n)
{
  if (!(p >= 0.0 && p <= 1.0)) return NAN;
  if (k >= n) return 0.0;
  if (p == 0.0) return 0.0;
  if (p == 1.0) return 1.0;
  const double odds = p / (1.0 - p);
  const double mode = (double)(n + 1) * p;
  if ((double)(k + 1) >= mode) {
    /* upper tail: terms decrease from i = k+1 upwards */
    double t = exp(mm_shim_binom_logpmf(k + 1, p, n));
    double sum = 0.0;
    for (unsigned int i = k + 1; i <= n; i++) {
      sum += t;
      if (t < sum * 1e-18) break;
      t *= odds * (double)(n - i) / (double)(i + 1);
    }
    return sum > 1.0 ? 1.0 : sum;
  } else {
    /* lower tail P(X <= k): terms decrease from i = k downwards */
    double t = exp(mm_shim_binom_logpmf(k, p, n));
    double sum = 0.0;
    for (unsigned int i = k;; i--) {
      sum += t;
      if (i == 0 || t < sum * 1e-18) break;
      t *= (double)i / (odds * (double)(n - i + 1));
    }
    double q = 1.0 - sum;
    return q < 0.0 ? 0.0 : q;
  }
}

/* P(k) for k successes in t draws without replacement from n1 successes, n2 failures */
static inline double gsl_ran_hypergeometric_pdf(const unsigned int k, const unsigned int n1,
                                                const unsigned int n2, unsigned int t)
{
  if (t > n1 + n2) t = n1 + n2;
  if (k > n1 || k > t) return 0.0;
  if (t > n2 && k + n2 < t) return 0.0;
  double c1 = mm_shim_lnchoose(n1, k);
  double c2 = mm_shim_lnchoose(n2, t - k);
  double c3 = mm_shim_lnchoose(n1 + n2, t);
  return exp(c1 + c2 - c3);
}

/* P(X <= k) for the same distribution */
static inline double gsl_cdf_hypergeometric_P(const unsigned int k, const unsigned int n1,
                                              const unsigned int n2, const unsigned int t)
{
  if (t > n1 + n2) return NAN;
  unsigned int lo = (t > n2) ? t - n2 : 0;
  unsigned int hi = (t < n1) ? t : n1;
  if (k >= hi) return 1.0;
  if (k < lo) return 0.0;
  /* sum the pmf from lo..k with the exact term ratio; start term by log-gamma. Terms below e^-700 are skipped in log
   * space: a subnormal start term has too few significant bits, and the recurrence would carry its error into every
   * term after it (at sketch size 1000 this moved cut-offs by up to 4) */
  double lt = mm_shim_lnchoose(n1, lo) + mm_shim_lnchoose(n2, t - lo) - mm_shim_lnchoose(n1 + n2, t);
  unsigned int i = lo;
  for (; i <= k && lt < -700.0; i++)
    lt += log(((double)(n1 - i) * (double)(t - i)) / ((double)(i + 1) * (double)(n2 - t + i + 1)));
  double term = exp(lt);
  double sum = 0.0;
  for (; i <= k; i++) {
    sum += term;
    term *= ((double)(n1 - i) * (double)(t - i)) /
            ((double)(i + 1) * (double)(n2 - t + i + 1));
  }
  return sum > 1.0 ? 1.0 : sum;
}

#ifdef __cplusplus
}
#endif
#endif
