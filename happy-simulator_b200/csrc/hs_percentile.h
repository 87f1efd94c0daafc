/* hs_percentile.h -- p50 and p99 of a bucket's values (hs_set_bucket_percentiles), shared, from this ONE source, by
 *   - the sm_90a kernels (nvcc, __device__: hs_buckets.cuh), and
 *   - the CPU tests' ctypes twin (gcc, tests/bucket_pct_twin.c),
 * as hs_sampler.h is shared.
 *
 * The reference (instrumentation/data.py:197-210, _percentile_sorted(sorted(vals), p)) sorts the bucket's values and
 * interpolates:  pos = p * (n - 1),  lo = int(pos),  hi = min(lo + 1, n - 1),  frac = pos - lo,
 *                vals[lo] * (1.0 - frac) + vals[hi] * frac.
 * Only the four order statistics lo50, hi50, lo99, hi99 are needed, so the values are not sorted: an in-place
 * selection puts the lo99-th smallest at index lo99 with everything smaller before it, the lo50-th is selected
 * among those, and each hi is the minimum of what lies above its lo.  Equal values have equal bits here (the values
 * are finite and non-negative: latencies, Probe metrics), so any correct selection returns the reference's operands.
 * Every operation of the interpolation is explicitly rounded (HS_MUL / HS_SUB / HS_ADD): the last line must not be
 * contracted into an FMA. */
#ifndef HS_PERCENTILE_H
#define HS_PERCENTILE_H

#include "hs_sampler.h"

/* Move the k-th smallest (0-based, k < n) of v[0 .. n) to v[k], with v[i] <= v[k] for i < k and v[i] >= v[k] for
 * i > k (Hoare's FIND in Wirth's form; the pivot is the median of the range's first, middle and last values, so a
 * sorted or reversed range halves at every pass). */
HS_HD void hs_pct_select(double *v, uint32_t n, uint32_t k)
{
    int32_t l = 0, m = (int32_t)n - 1;
    const int32_t kk = (int32_t)k;
    while (l < m) {
        const double a = v[l], b = v[(l + m) >> 1], c = v[m];
        const double x = (a < b) ? ((b < c) ? b : (a < c) ? c : a) : ((a < c) ? a : (b < c) ? c : b);
        int32_t i = l, j = m;
        do {
            while (v[i] < x) i++;
            while (x < v[j]) j--;
            if (i <= j) { const double t = v[i]; v[i] = v[j]; v[j] = t; i++; j--; }
        } while (i <= j);
        if (j < kk) l = i;
        if (kk < i) m = j;
    }
}

/* min of v[a .. b), a < b */
HS_HD double hs_pct_min(const double *v, uint32_t a, uint32_t b)
{
    double x = v[a];
    for (uint32_t i = a + 1; i < b; ++i) x = (v[i] < x) ? v[i] : x;
    return x;
}

/* the reference's interpolation between the order statistics at lo and lo + 1 (clamped) */
HS_HD double hs_pct_interp(double vlo, double vhi, double frac)
{
    return HS_ADD(HS_MUL(vlo, HS_SUB(1.0, frac)), HS_MUL(vhi, frac));
}

/* pos = p * (n - 1) and lo = int(pos) */
HS_HD uint32_t hs_pct_lo(double p, uint32_t n, double *pos)
{
    *pos = HS_MUL(p, HS_LL2D((long long)(n - 1u)));
    return (uint32_t)HS_D2LL(*pos);
}

/* out[0] = _percentile_sorted(sorted(v), 0.50), out[1] = _percentile_sorted(sorted(v), 0.99) of v[0 .. n), n >= 1.
 * Permutes v. */
HS_HD void hs_bucket_percentiles(double *v, uint32_t n, double *out)
{
    double pos99, pos50;
    const uint32_t lo99 = hs_pct_lo(0.99, n, &pos99), lo50 = hs_pct_lo(0.50, n, &pos50);
    hs_pct_select(v, n, lo99);                          /* v[0 .. lo99] = the lo99 + 1 smallest, v[lo99] the largest of them */
    const double l99 = v[lo99];
    const double h99 = (lo99 + 1u < n) ? hs_pct_min(v, lo99 + 1u, n) : l99;
    double l50, h50;
    if (lo50 == lo99) { l50 = l99; h50 = h99; }
    else {                                              /* lo50 < lo99: both of its statistics lie in v[0 .. lo99] */
        hs_pct_select(v, lo99 + 1u, lo50);
        l50 = v[lo50];
        h50 = hs_pct_min(v, lo50 + 1u, lo99 + 1u);
    }
    out[0] = hs_pct_interp(l50, h50, HS_SUB(pos50, HS_LL2D((long long)lo50)));
    out[1] = hs_pct_interp(l99, h99, HS_SUB(pos99, HS_LL2D((long long)lo99)));
}

#endif /* HS_PERCENTILE_H */
