/* hs_buckets.cuh -- time buckets of the Sink / Probe samples (hs_set_buckets, include/hs_b200.h).
 *
 * What the reference computes on the host from a replica's complete sample list, Data.bucket(window_s)
 * (instrumentation/data.py:127-158: per bucket count, sum(), max(); mean = sum / count), accumulated on the device as
 * the samples arrive, so that an ensemble gets every replica's curve without materialising its samples.  A replica's
 * samples come in time order, so each bucketed row only ever adds to its CURRENT bucket: the row's accumulator
 * (hs_bucket_acc: the bucket's index, count, Neumaier pair and max) lives in the replica's state -- registers in the lane
 * engine, a slot per row in the replica block of the thread engine (HBM, cached in L1 like the entity cells) and of the
 * warp engine (staged in shared memory) -- and a sample costs one compare and the update.  The 32-byte record in HBM is
 * written when the row moves on to another bucket and, for every row, when the launch ends: at the end of the run and
 * at a window pause.  An accumulator starts every launch empty and takes up its first bucket from the record (zeros,
 * or what an earlier window left there), so a run cut into windows gives the uncut run's records.
 *
 * The engines call hs_bucket_add only from their HS_LF_BUCKETS / HS_WF_BUCKETS instantiations; every other kernel is
 * compiled without it.  Then a deterministic two-stage reduction per sweep cell (as hs_totals.cuh): no float atomics,
 * a fixed summation order.
 *
 * Percentiles (hs_set_bucket_percentiles; the HS_LF_BUCKET_PCT / HS_WF_BUCKET_PCT instantiations, which get
 * hs_bucket_pct_args): p50 and p99 need the bucket's values, but only the current bucket's.  Each (replica, row) has a
 * buffer of `cap` doubles in HBM, separate from the replica block (the warp engine stages that in shared memory);
 * hs_bucket_add stores a sample at index count (before the increment), and every flush of the record also selects
 * the percentiles of the `count` buffered values (hs_percentile.h) into pct[replica][row][slot].  Selection permutes
 * the buffer, which is harmless: a resumed window only appends to the same multiset, at index count, and the next
 * flush selects again.  A bucket with more than cap samples gets NaN and its replica HS_ST_BUCKET_OVERFLOW. */
#ifndef HS_BUCKETS_CUH
#define HS_BUCKETS_CUH

#include "hs_sampler.h"
#include "hs_percentile.h"
#include "../../include/hs_b200.h"

#define HS_BUCKET_SLICE 256u        /* replicas per first-stage slice of the cell reduction */

/* The bucket arguments reach every engine kernel (lane, warp, both thread forms) as its last parameter, of type
 * hs_bucket_args in the bucket instantiations and of the empty hs_no_bucket_args in every other one, an unused
 * parameter that changes none of their code. */
struct hs_bucket_args {
    double w;                       /* width in seconds */
    uint32_t n, rows;               /* buckets per row, bucketed rows (SINK and PROBE rows) */
    hs_bucket *rec;                 /* [replica][rows][n + 1] */
    int64_t *past_end;              /* [replica][rows]: index of the samples in slot n */
    uint32_t acc_off, pad;          /* thread / warp engine: byte offset of the rows' accumulators in a replica block */
};
/* ... and of the percentile instantiations */
struct hs_bucket_pct_args : hs_bucket_args {
    double *vals;                   /* [replica][rows][cap]: the values of each row's current bucket */
    double2 *pct;                   /* [replica][rows][n + 1]: {p50, p99} of every bucket (NaN, NaN: more than cap samples) */
    uint32_t *status;               /* [replica]: HS_ST_BUCKET_OVERFLOW once a bucket overflowed, else 0 */
    uint32_t cap, pad2;             /* values per buffer */
};
struct hs_no_bucket_args {};
template <bool ON, bool PCT = false> struct hs_bucket_args_of { typedef hs_no_bucket_args type; };
template <> struct hs_bucket_args_of<true, false> { typedef hs_bucket_args type; };
template <> struct hs_bucket_args_of<true, true> { typedef hs_bucket_pct_args type; };

/* a row's current bucket: k = its index (< 0: none yet in this launch), b = its record so far.  40 bytes */
struct hs_bucket_acc { double k; hs_bucket b; };
struct hs_no_bucket_acc {};

/* Data.bucket's index of a sample at `ns`: math.floor(t / window_s) with t = Instant.to_seconds() -- the correctly
 * rounded ns / 1e9, then a correctly rounded division by the width, then floor.  (Integer arithmetic on ns is a
 * different function: 300 000 000 ns at w = 0.1 is bucket 2, because 0.3 / 0.1 == 2.9999999999999996.) */
__device__ __forceinline__ double hs_bucket_index(int64_t ns, double w) { return floor(HS_DIV(hs_ns_to_seconds(ns), w)); }

/* the index of bucket k of row `row` of replica r among the records (k >= n: slot n) */
__device__ __forceinline__ size_t hs_bucket_slot_index(const hs_bucket_args &BK, uint32_t r, uint32_t row, double k)
{
    return ((size_t)r * BK.rows + row) * (BK.n + 1u) + (k < (double)BK.n ? (uint32_t)k : BK.n);
}
__device__ __forceinline__ hs_bucket *hs_bucket_slot(const hs_bucket_args &BK, uint32_t r, uint32_t row, double k)
{
    return BK.rec + hs_bucket_slot_index(BK, r, row, k);
}

/* percentiles: nothing in the instantiations without them */
__device__ __forceinline__ void hs_bucket_keep(const hs_bucket_args &, uint32_t, uint32_t, const hs_bucket_acc &, double) {}
__device__ __forceinline__ void hs_bucket_pct_flush(const hs_bucket_args &, uint32_t, uint32_t, const hs_bucket_acc &) {}

/* the sample's value into the buffer of its row, at index count (nothing past cap: the flush reports the overflow) */
__device__ __forceinline__ void hs_bucket_keep(const hs_bucket_pct_args &BK, uint32_t r, uint32_t row, const hs_bucket_acc &a,
                                               double v)
{
    if (a.b.count < (int64_t)BK.cap) BK.vals[((size_t)r * BK.rows + row) * BK.cap + (size_t)a.b.count] = v;
}

/* p50 and p99 of the buffered values of a row's bucket into its percentile record.  Not inlined: it runs once per
 * bucket, and the engines' event loops keep their registers */
__device__ __noinline__ void hs_bucket_pct_store(const hs_bucket_pct_args &BK, uint32_t r, uint32_t row, double k, int64_t count)
{
    double2 q;
    if (count > (int64_t)BK.cap) {
        q.x = q.y = __longlong_as_double(0x7ff8000000000000LL);
        BK.status[r] = HS_ST_BUCKET_OVERFLOW;
    } else {
        double o[2];
        hs_bucket_percentiles(BK.vals + ((size_t)r * BK.rows + row) * BK.cap, (uint32_t)count, o);
        q.x = o[0]; q.y = o[1];
    }
    BK.pct[hs_bucket_slot_index(BK, r, row, k)] = q;
}
__device__ __forceinline__ void hs_bucket_pct_flush(const hs_bucket_pct_args &BK, uint32_t r, uint32_t row, const hs_bucket_acc &a)
{
    hs_bucket_pct_store(BK, r, row, a.k, a.b.count);
}

/* store a row's accumulator into its record, and its percentiles into theirs (nothing if it holds no bucket).
 * BA: hs_bucket_args or hs_bucket_pct_args */
template <class BA>
__device__ __forceinline__ void hs_bucket_flush(const BA &BK, uint32_t r, uint32_t row, const hs_bucket_acc &a)
{
    if (a.k < 0.0) return;
    if (a.k >= (double)BK.n) BK.past_end[(size_t)r * BK.rows + row] = (int64_t)a.k;   /* past end_ns: hs_run's check leaves
                                                                                          one event there */
    *hs_bucket_slot(BK, r, row, a.k) = a.b;
    hs_bucket_pct_flush(BK, r, row, a);
}

/* one sample of bucketed row `row` of replica r: value v at ns, into the row's accumulator a */
template <class BA>
__device__ __forceinline__ void hs_bucket_add(const BA &BK, uint32_t r, uint32_t row, hs_bucket_acc &a, int64_t ns, double v)
{
    const double k = hs_bucket_index(ns, BK.w);
    if (k != a.k) {                 /* the row moves on: the finished bucket goes to HBM, the new one starts from its record */
        hs_bucket_flush(BK, r, row, a);
        a.k = k;
        a.b = *hs_bucket_slot(BK, r, row, k);
    }
    hs_bucket_keep(BK, r, row, a, v);
    a.b.max = (a.b.count == 0 || v > a.b.max) ? v : a.b.max;           /* max(): the first of equal values */
    a.b.count++;
    hs_neumaier_add(&a.b.sum, &a.b.comp, v);
}

/* general engines: the rows' accumulators in the replica block `blk`; empty at the start of a launch, stored at its end */
__device__ __forceinline__ hs_bucket_acc *hs_bucket_accs(const hs_bucket_args &BK, unsigned char *blk)
{
    return (hs_bucket_acc *)(blk + BK.acc_off);
}
__device__ __forceinline__ void hs_bucket_begin(const hs_bucket_args &BK, hs_bucket_acc *a)
{
    for (uint32_t b = 0; b < BK.rows; ++b) a[b].k = -1.0;
}
template <class BA>
__device__ __forceinline__ void hs_bucket_end(const BA &BK, uint32_t r, const hs_bucket_acc *a)
{
    for (uint32_t b = 0; b < BK.rows; ++b) hs_bucket_flush(BK, r, b, a[b]);
}
/* the replica's status bits from its buckets (after the launch's last flush) */
__device__ __forceinline__ uint32_t hs_bucket_status(const hs_bucket_pct_args &BK, uint32_t r) { return BK.status[r]; }
__device__ __forceinline__ uint32_t hs_bucket_status(const hs_bucket_args &, uint32_t) { return 0u; }
__device__ __forceinline__ uint32_t hs_bucket_status(const hs_no_bucket_args &, uint32_t) { return 0u; }

/* the instantiations without buckets: no state and no calls (their FLAGS tests are false); these only let them compile */
__device__ __forceinline__ void hs_bucket_add(const hs_no_bucket_args &, uint32_t, uint32_t, hs_no_bucket_acc &, int64_t, double) {}
__device__ __forceinline__ void hs_bucket_add(const hs_no_bucket_args &, uint32_t, uint32_t, hs_no_bucket_acc *, int64_t, double) {}
__device__ __forceinline__ hs_no_bucket_acc *hs_bucket_accs(const hs_no_bucket_args &, unsigned char *) { return nullptr; }
__device__ __forceinline__ void hs_bucket_begin(const hs_no_bucket_args &, hs_no_bucket_acc *) {}
__device__ __forceinline__ void hs_bucket_end(const hs_no_bucket_args &, uint32_t, const hs_no_bucket_acc *) {}
__device__ __forceinline__ void hs_bucket_flush(const hs_no_bucket_args &, uint32_t, uint32_t, const hs_no_bucket_acc &) {}
template <class BA>
__device__ __forceinline__ void hs_bucket_add(const BA &BK, uint32_t r, uint32_t row, hs_bucket_acc *a, int64_t ns, double v)
{
    hs_bucket_add(BK, r, row, a[row], ns, v);
}
__device__ __forceinline__ void hs_bucket_reset(hs_bucket_acc &a) { a.k = -1.0; }
__device__ __forceinline__ void hs_bucket_reset(hs_no_bucket_acc &) {}
template <bool ON> struct hs_bucket_acc_of { typedef hs_no_bucket_acc type; };
template <> struct hs_bucket_acc_of<true> { typedef hs_bucket_acc type; };

/* ---- per-cell reduction ------------------------------------------------------------------------------------- */

struct hs_bucket_slice { uint32_t begin, end; };    /* replicas [begin, end) of one cell, in index order */

/* What the two stages fold: a source (the per-replica data, addressed by record index) into a total.  The records
 * give hs_bucket_total; the records with their percentiles give hs_bucket_pct_total. */
struct hs_bucket_src { const hs_bucket *__restrict__ b; };
struct hs_bucket_pct_src { const hs_bucket *__restrict__ b; const double2 *__restrict__ pct; };

__device__ __forceinline__ void hs_bucket_total_zero(hs_bucket_total &t)
{
    t.replicas = 0; t.count = 0; t.sum = 0.0; t.mean_sum = 0.0; t.mean_sq_sum = 0.0;
    t.max = __longlong_as_double(0xfff0000000000000LL);
}

/* one replica's bucket: its sum as sum() returns it, its mean as Data.bucket computes it */
__device__ __forceinline__ void hs_bucket_total_add(hs_bucket_total &t, const hs_bucket_src &src, size_t i)
{
    const hs_bucket b = src.b[i];
    if (b.count == 0) return;
    const double s = hs_neumaier_result(b.sum, b.comp);
    const double m = HS_DIV(s, (double)b.count);
    t.replicas += 1; t.count += b.count;
    t.sum = HS_ADD(t.sum, s);
    t.mean_sum = HS_ADD(t.mean_sum, m);
    t.mean_sq_sum = HS_ADD(t.mean_sq_sum, HS_MUL(m, m));
    t.max = b.max > t.max ? b.max : t.max;
}

__device__ __forceinline__ void hs_bucket_total_merge(hs_bucket_total &a, const hs_bucket_total &b)
{
    a.replicas += b.replicas; a.count += b.count;
    a.sum = HS_ADD(a.sum, b.sum);
    a.mean_sum = HS_ADD(a.mean_sum, b.mean_sum);
    a.mean_sq_sum = HS_ADD(a.mean_sq_sum, b.mean_sq_sum);
    a.max = b.max > a.max ? b.max : a.max;
}

__device__ __forceinline__ void hs_bucket_total_zero(hs_bucket_pct_total &t)
{
    t.p50_sum = 0.0; t.p50_sq_sum = 0.0; t.p99_sum = 0.0; t.p99_sq_sum = 0.0;
}

/* one replica's bucket percentiles, if the bucket has samples */
__device__ __forceinline__ void hs_bucket_total_add(hs_bucket_pct_total &t, const hs_bucket_pct_src &src, size_t i)
{
    if (src.b[i].count == 0) return;
    const double2 q = src.pct[i];
    t.p50_sum = HS_ADD(t.p50_sum, q.x);
    t.p50_sq_sum = HS_ADD(t.p50_sq_sum, HS_MUL(q.x, q.x));
    t.p99_sum = HS_ADD(t.p99_sum, q.y);
    t.p99_sq_sum = HS_ADD(t.p99_sq_sum, HS_MUL(q.y, q.y));
}

__device__ __forceinline__ void hs_bucket_total_merge(hs_bucket_pct_total &a, const hs_bucket_pct_total &b)
{
    a.p50_sum = HS_ADD(a.p50_sum, b.p50_sum);
    a.p50_sq_sum = HS_ADD(a.p50_sq_sum, b.p50_sq_sum);
    a.p99_sum = HS_ADD(a.p99_sum, b.p99_sum);
    a.p99_sq_sum = HS_ADD(a.p99_sq_sum, b.p99_sq_sum);
}

/* stage 1: partial[s][j] = slice s's replicas folded in index order, j = row * (n + 1) + bucket (one thread per j:
 * neighbouring threads read neighbouring records of the same replica) */
template <class Src, class T>
__global__ void __launch_bounds__(128)
hs_bucket_partial_kernel(const Src src, uint32_t per_replica, const hs_bucket_slice *__restrict__ slices,
                         uint32_t n_slices, T *__restrict__ partial)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= per_replica) return;
    for (uint32_t s = blockIdx.y; s < n_slices; s += gridDim.y) {
        const hs_bucket_slice sl = slices[s];
        T t; hs_bucket_total_zero(t);
        for (uint32_t r = sl.begin; r < sl.end; ++r) hs_bucket_total_add(t, src, (size_t)r * per_replica + j);
        partial[(size_t)s * per_replica + j] = t;
    }
}

/* stage 2: out[c][j] = the slices of cell c (cell_first[c] .. cell_first[c + 1] in cell_slices, ascending) folded in order */
template <class T>
__global__ void __launch_bounds__(128)
hs_bucket_final_kernel(const T *__restrict__ partial, uint32_t per_replica, const uint32_t *__restrict__ cell_first,
                       const uint32_t *__restrict__ cell_slices, uint32_t n_cells, T *__restrict__ out)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= per_replica) return;
    for (uint32_t c = blockIdx.y; c < n_cells; c += gridDim.y) {
        T t; hs_bucket_total_zero(t);
        for (uint32_t k = cell_first[c]; k < cell_first[c + 1]; ++k)
            hs_bucket_total_merge(t, partial[(size_t)cell_slices[k] * per_replica + j]);
        out[(size_t)c * per_replica + j] = t;
    }
}

#endif /* HS_BUCKETS_CUH */
