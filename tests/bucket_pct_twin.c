/* ctypes twin of hs_percentile.h (test infrastructure): the selection and interpolation the kernels run for bucket
 * percentiles, compiled by gcc from the same header, so the CPU tests can hold them against the reference's
 * _percentile_sorted.  Built by tests/bucket_pct_lib.py with -ffp-contract=off, as the oracle is. */
#include <stdint.h>

#include "../happy-simulator_b200/csrc/hs_percentile.h"

/* m multisets packed in v: multiset k is v[off[k] .. off[k + 1]), each at least one value; out[2k] = p50, out[2k + 1]
 * = p99.  Permutes v, as the device permutes its buffers. */
void hs_cpu_bucket_percentiles(double *v, const uint64_t *off, uint32_t m, double *out)
{
    for (uint32_t k = 0; k < m; ++k)
        hs_bucket_percentiles(v + off[k], (uint32_t)(off[k + 1] - off[k]), out + 2 * (uint64_t)k);
}
