/* hs_sampler.h -- counter-based RNG, natural log and int-ns/float-seconds time
 * arithmetic shared, from this ONE source, by
 *   - the sm_90a kernels (nvcc, __device__),
 *   - the CPU oracle in oracle/ (gcc), and
 *   - the ctypes twins (hs_cpu_*) that the Philox plug-ins call when they are
 *     injected into the unmodified reference (tests/golden/gen_golden.py).
 * Sharing the source is what makes "bit-exact on the same seeds" a construction
 * and not a probability (SURVEY.md section 7, "log parity").
 *
 * Every floating-point operation below is an explicitly rounded IEEE-754
 * binary64 operation.  Nothing here may be contracted or reassociated by a
 * compiler: on the device the __dadd_rn/__dmul_rn/__fma_rn/__ddiv_rn intrinsics
 * are never contracted; on the host the translation unit must be compiled with
 * -ffp-contract=off (the oracle Makefile does) and fma() is the correctly
 * rounded libm/hardware fma.
 *
 * Reference arithmetic restated here (paths relative to /root/reference):
 *   T1  Instant/Duration.from_seconds : int(seconds * 1e9), truncation toward 0
 *       happysimulator/core/temporal.py:58-62,201-205
 *   T2  Instant.__add__(float)        : ns + int(other * 1e9)
 *       happysimulator/core/temporal.py:213-223
 *   T3  to_seconds                    : float(ns) / 1e9
 *       happysimulator/core/temporal.py:66-68,209-211
 *   L2  ArrivalTimeProvider.next_arrival_time fast path
 *       happysimulator/load/arrival_time_provider.py:70-78
 *   L3  PoissonArrivalTimeProvider._get_target_integral_value: -log(1.0 - U)
 *       happysimulator/load/providers/poisson_arrival.py:31
 *   D1  ExponentialLatency.get_latency: expovariate(l) = -log(1.0 - U) / l,
 *       l = 1 / mean;  happysimulator/distributions/exponential.py:36,43-45
 */
#ifndef HS_SAMPLER_H
#define HS_SAMPLER_H

#include <stdint.h>

#if defined(__CUDA_ARCH__)
#define HS_HD __host__ __device__ __forceinline__
#define HS_ADD(a, b) __dadd_rn((a), (b))
#define HS_SUB(a, b) __dadd_rn((a), -(b))
#define HS_MUL(a, b) __dmul_rn((a), (b))
#define HS_DIV(a, b) __ddiv_rn((a), (b))
#define HS_FMA(a, b, c) __fma_rn((a), (b), (c))
#define HS_SQRT(a) __dsqrt_rn((a))
#define HS_D2LL(x) __double2ll_rz(x)
#define HS_LL2D(x) __ll2double_rn(x)
#define HS_MULHI32(a, b) __umulhi((a), (b))
#define HS_D2BITS(x) ((uint64_t)__double_as_longlong(x))
#define HS_BITS2D(x) __longlong_as_double((long long)(x))
#else
#include <math.h>
#include <string.h>
#if defined(__CUDACC__)
#define HS_HD __host__ __device__ inline
#else
#define HS_HD static inline
#endif
#define HS_ADD(a, b) ((a) + (b))
#define HS_SUB(a, b) ((a) - (b))
#define HS_MUL(a, b) ((a) * (b))
#define HS_DIV(a, b) ((a) / (b))
#define HS_FMA(a, b, c) fma((a), (b), (c))
#define HS_SQRT(a) sqrt((a))              /* IEEE correctly rounded, like math.sqrt */
#define HS_D2LL(x) ((long long)(x))
#define HS_LL2D(x) ((double)(long long)(x))
#define HS_MULHI32(a, b) ((uint32_t)(((uint64_t)(a) * (uint64_t)(b)) >> 32))
static inline uint64_t hs_d2bits_(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }
static inline double hs_bits2d_(uint64_t u) { double x; memcpy(&x, &u, 8); return x; }
#define HS_D2BITS(x) hs_d2bits_(x)
#define HS_BITS2D(x) hs_bits2d_(x)
#endif

/* ------------------------------------------------------------------------ */
/* Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as
 * easy as 1, 2, 3", SC'11).  Key = 64-bit run seed; counter =
 * (draw_pair lo, draw_pair hi, replica id, stream id).                      */

#define HS_PHILOX_M0 0xD2511F53u
#define HS_PHILOX_M1 0xCD9E8D57u
#define HS_PHILOX_W0 0x9E3779B9u
#define HS_PHILOX_W1 0xBB67AE85u

typedef struct { uint32_t x, y, z, w; } hs_u32x4;

HS_HD hs_u32x4 hs_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                uint32_t k0, uint32_t k1)
{
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = HS_MULHI32(HS_PHILOX_M0, c0), lo0 = HS_PHILOX_M0 * c0;
        uint32_t hi1 = HS_MULHI32(HS_PHILOX_M1, c2), lo1 = HS_PHILOX_M1 * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += HS_PHILOX_W0; k1 += HS_PHILOX_W1;
    }
    hs_u32x4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
    return o;
}

/* Stream ids (SURVEY.md section 8(d)). */
#define HS_STREAM_ARRIVAL 0u
#define HS_STREAM_SERVICE 1u
#define HS_STREAM_ROUTING 2u
#define HS_STREAM_LINK_LOSS 3u      /* WindowedCoordinator._rng.random(), coordinator.py:204 */
#define HS_STREAM_LINK_LATENCY 4u   /* PartitionLink.latency.sample(), coordinator.py:209 (| latency object id << 8) */

/* 53-bit uniform in [0,1) from two 32-bit words, the genrand_res53 recipe both
 * reference generators use (CPython random.random(), numpy legacy
 * random_sample): (a>>5, b>>6) -> (a*2^26 + b) / 2^53.                      */
HS_HD double hs_u53(uint32_t a, uint32_t b)
{
    uint64_t m = ((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6);
    return HS_MUL(HS_LL2D((long long)m), 1.1102230246251565e-16); /* 2^-53, exact */
}

/* One Philox block yields the two uniforms draw 2p and draw 2p+1 of a stream.
 * The stream id word also carries the entity index (server / source) so that
 * every consumer owns an independent stream: sid = stream | (entity << 8).   */
HS_HD void hs_uniform_pair(uint64_t seed, uint32_t replica, uint32_t sid, uint64_t pair,
                           double *u0, double *u1)
{
    hs_u32x4 r = hs_philox4x32_10((uint32_t)pair, (uint32_t)(pair >> 32), replica, sid,
                                  (uint32_t)seed, (uint32_t)(seed >> 32));
    *u0 = hs_u53(r.x, r.y);
    *u1 = hs_u53(r.z, r.w);
}

HS_HD double hs_uniform(uint64_t seed, uint32_t replica, uint32_t sid, uint64_t draw)
{
    double u0, u1;
    hs_uniform_pair(seed, replica, sid, draw >> 1, &u0, &u1);
    return (draw & 1u) ? u1 : u0;
}

/* Routing key of a request: SimpleEventProvider's context_fn draws client_id from a value distribution over
 * 0..n-1.  Uniform: int(u * n).  Zipf: bisect.bisect_left(cum_probs, u) clamped to n - 1 (distributions/
 * zipf.py:112-123), cum_probs computed by the host with the reference's arithmetic.                        */
HS_HD int32_t hs_routing_key(double u, int32_t n, const double *cum_probs)
{
    if (!cum_probs) return (int32_t)HS_D2LL(HS_MUL(u, (double)n));
    int32_t lo = 0, hi = n;                      /* bisect_left: first index with cum_probs[i] >= u */
    while (lo < hi) { const int32_t mid = (lo + hi) >> 1; if (cum_probs[mid] < u) lo = mid + 1; else hi = mid; }
    return lo < n - 1 ? lo : n - 1;
}

/* ------------------------------------------------------------------------ */
/* Natural logarithm for finite x > 0 (the sampler only ever passes
 * x = 1 - U in [2^-53, 1]).  Classic argument reduction x = 2^k (1+f),
 * sqrt(2)/2 <= 1+f < sqrt(2); s = f/(2+f); log(1+f) = 2s + s*R(s^2) with the
 * degree-7 minimax R of Sun's freely distributable fdlibm e_log.c
 * (error < 1 ulp).  Evaluated with explicitly rounded operations only, so the
 * device and the host produce the same bits.                                 */
HS_HD double hs_log(double x)
{
    const double ln2_hi = 6.93147180369123816490e-01; /* 0x3fe62e42fee00000 */
    const double ln2_lo = 1.90821492927058770002e-10; /* 0x3dea39ef35793c76 */
    const double Lg1 = 6.666666666666735130e-01;
    const double Lg2 = 3.999999999940941908e-01;
    const double Lg3 = 2.857142874366239149e-01;
    const double Lg4 = 2.222219843214978396e-01;
    const double Lg5 = 1.818357216161805012e-01;
    const double Lg6 = 1.531383769920937332e-01;
    const double Lg7 = 1.479819860511658591e-01;

    uint64_t ix = HS_D2BITS(x);
    int k = 0;
    if ((ix >> 52) == 0) {            /* subnormal: scale by 2^54 (never hit by 1-U) */
        x = HS_MUL(x, 18014398509481984.0);
        ix = HS_D2BITS(x);
        k = -54;
    }
    k += (int)(ix >> 52) - 1023;
    uint64_t man = ix & 0x000fffffffffffffULL;
    /* mantissa >= sqrt(2) -> halve it and bump the exponent */
    if (man >= 0x6a09e667f3bcdULL) { k += 1; ix = man | 0x3fe0000000000000ULL; }
    else                           {         ix = man | 0x3ff0000000000000ULL; }
    double f = HS_SUB(HS_BITS2D(ix), 1.0);
    double dk = HS_LL2D((long long)k);

    double s = HS_DIV(f, HS_ADD(2.0, f));
    double z = HS_MUL(s, s);
    double w = HS_MUL(z, z);
    double t1 = HS_MUL(w, HS_FMA(w, HS_FMA(w, Lg6, Lg4), Lg2));
    double t2 = HS_MUL(z, HS_FMA(w, HS_FMA(w, HS_FMA(w, Lg7, Lg5), Lg3), Lg1));
    double R = HS_ADD(t2, t1);
    double hfsq = HS_MUL(0.5, HS_MUL(f, f));
    /* log(x) = k*ln2_hi - ((hfsq - (s*(hfsq+R) + k*ln2_lo)) - f) */
    double inner = HS_FMA(s, HS_ADD(hfsq, R), HS_MUL(dk, ln2_lo));
    return HS_SUB(HS_MUL(dk, ln2_hi), HS_SUB(HS_SUB(hfsq, inner), f));
}

/* L3: exponential(1) target area, -log(1.0 - U). */
HS_HD double hs_exp1(double u) { return -hs_log(HS_SUB(1.0, u)); }

/* ------------------------------------------------------------------------ */
/* Time arithmetic (T1-T3, L2, D1).                                           */
#define HS_NS_PER_S 1000000000.0

HS_HD int64_t hs_seconds_to_ns(double seconds)          /* T1 */
{ return (int64_t)HS_D2LL(HS_MUL(seconds, HS_NS_PER_S)); }

/* Correctly rounded x / b for a divisor whose correctly rounded reciprocal y = RN(1/b) is at hand:
 *     q = RN(x * y);   r = x - q * b  (exact in one fma: q is a faithful quotient);   x / b = RN(q + r * y)
 * (Markstein, "Computation of elementary functions on the IBM RISC System/6000 processor", IBM J. Res.
 * Dev. 34 (1990), Theorem 8.5 -- the final step of every fma-based IEEE division, including the one nvcc
 * emits for `/`; valid while no intermediate over-/underflows, which the magnitudes on this path -- ns
 * counts below 2^63, targets in [2^-53, 37], rates in [1e-6, 1e12] -- never approach).  Three fp64
 * instructions instead of the ~20 of a general division; the result is bit-identical to `x / b`
 * (tests/test_sampler.py checks it against the C division on random and structured operands,
 * tools/divcheck.c ran 5e9 more).  The sign of a zero quotient is not preserved (-0.0 / b gives +0.0);
 * no caller can observe it: the quotients are added to a non-negative time or truncated to an integer. */
HS_HD double hs_div_recip(double x, double b, double y)
{
    const double q = HS_MUL(x, y);
    const double r = HS_FMA(-q, b, x);
    return HS_FMA(r, y, q);
}
#define HS_NS_PER_S_RECIP 1e-9      /* the double nearest 10^-9 = RN(1 / 1e9) */

/* For run-time divisors (a Source's rate, a server's lambda) the caller passes y = 1.0 / b, or 0.0 to ask for
 * the general division: for divisors outside the comfortable range and for a significand of all ones,
 * the one case the literature singles out for reciprocal-based division. */
HS_HD int hs_recip_divisor_ok(double b)
{
    const uint64_t u = HS_D2BITS(b);
    const uint64_t man = u & 0x000fffffffffffffULL;
    return b >= 1e-100 && b <= 1e100 && man != 0x000fffffffffffffULL;
}
HS_HD double hs_div_by(double x, double b, double y)
{ return y != 0.0 ? hs_div_recip(x, b, y) : HS_DIV(x, b); }

HS_HD double hs_ns_to_seconds(int64_t ns)               /* T3 */
{ return hs_div_recip(HS_LL2D(ns), HS_NS_PER_S, HS_NS_PER_S_RECIP); }

/* L2: next arrival of a constant-rate profile; target = 1.0 (constant
 * provider) or hs_exp1(u) (Poisson provider). */
HS_HD int64_t hs_next_arrival_ns(int64_t cur_ns, double target, double rate)
{
    double t_next = HS_ADD(hs_ns_to_seconds(cur_ns), HS_DIV(target, rate));
    return hs_seconds_to_ns(t_next);
}

/* L2 with the rate's reciprocal precomputed by the caller (rate_recip = 1.0 / rate by IEEE division, or 0.0) */
HS_HD int64_t hs_next_arrival_ns_r(int64_t cur_ns, double target, double rate, double rate_recip)
{
    double t_next = HS_ADD(hs_ns_to_seconds(cur_ns), hs_div_by(target, rate, rate_recip));
    return hs_seconds_to_ns(t_next);
}

/* D1: ExponentialLatency.get_latency -> Duration (ns). lambda = 1/mean is
 * computed once by the caller exactly as the reference does (exponential.py:36). */
HS_HD int64_t hs_exp_latency_ns(double u, double lambda)
{ return hs_seconds_to_ns(HS_DIV(hs_exp1(u), lambda)); }
HS_HD int64_t hs_exp_latency_ns_r(double u, double lambda, double lambda_recip)
{ return hs_seconds_to_ns(hs_div_by(hs_exp1(u), lambda, lambda_recip)); }

/* Server.handle_queued_event: service_time_s = Duration.to_seconds(); the
 * generator yields it and ProcessContinuation adds int(delay*1e9) to now
 * (server/server.py:246-253, core/event.py:499, core/temporal.py:221-222).   */
HS_HD int64_t hs_resume_ns(int64_t now_ns, double delay_s)
{ return now_ns + hs_seconds_to_ns(delay_s); }

/* ------------------------------------------------------------------------ */
/* Sink.average_latency() is sum(latencies_s) / n (components/common.py:46-50) and
 * CPython >= 3.12 (the reference requires >= 3.13, pyproject.toml:11) evaluates
 * float sum() with Neumaier compensation (Python/bltinmodule.c, builtin_sum):
 *     t = s + x;  c += |s| >= |x| ? (s - t) + x : (x - t) + s;  s = t
 * and returns s + c when c is non-zero and finite.  Same steps here.          */
HS_HD void hs_neumaier_add(double *s, double *c, double x)
{
    double t = HS_ADD(*s, x);
    double as = *s < 0.0 ? -*s : *s, ax = x < 0.0 ? -x : x;
    if (as >= ax) *c = HS_ADD(*c, HS_ADD(HS_SUB(*s, t), x));
    else          *c = HS_ADD(*c, HS_ADD(HS_SUB(x, t), *s));
    *s = t;
}

HS_HD double hs_neumaier_result(double s, double c)
{
    /* "if (c && Py_IS_FINITE(c)) f_result += c" */
    uint64_t b = HS_D2BITS(c) & 0x7fffffffffffffffULL;
    if (b != 0 && b < 0x7ff0000000000000ULL) return HS_ADD(s, c);
    return s;
}

/* ------------------------------------------------------------------------ */
/* Latency histogram (instrumentation reduced on the device: at ensemble scale the
 * reference's per-request latency lists cannot be materialised, SURVEY.md section 7).
 * 64 log-spaced bins over the integer latency in ns, two bins per octave:
 *   bin 0: lat < 1024 ns;  bin 1 + 2 (e - 10) + m: lat in [2^e (1 + m/2), 2^e (1 + (m+1)/2)),
 *   e = floor(log2 lat) >= 10, m in {0, 1};  the last bin (63) also takes everything above.
 * Pure integer arithmetic, hence identical on every party.                          */
#define HS_HIST_BINS 64
HS_HD uint32_t hs_latency_bin(int64_t lat_ns)
{
    if (lat_ns < 1024) return 0u;
    uint64_t v = (uint64_t)lat_ns;
    int e = 0;
#if defined(__CUDA_ARCH__)
    e = 63 - __clzll((long long)v);
#else
    e = 63 - __builtin_clzll(v);
#endif
    const uint32_t m = (uint32_t)((v >> (e - 1)) & 1u);
    const uint32_t b = 1u + 2u * (uint32_t)(e - 10) + m;
    return b > 63u ? 63u : b;
}

/* ------------------------------------------------------------------------ */
/* Order hash over the processed-event sequence: FNV-1a style over the two
 * 64-bit words of the 16-byte event record (time_ns, idx | kind<<32 | ent<<40). */
#define HS_HASH_INIT 0xcbf29ce484222325ULL
#define HS_HASH_MUL  0x100000001b3ULL

HS_HD uint64_t hs_record_word1(uint64_t idx, uint32_t kind, uint32_t ent)
{ return (idx & 0xffffffffULL) | ((uint64_t)(kind & 0xffu) << 32) | ((uint64_t)(ent & 0xffffu) << 40); }

HS_HD uint64_t hs_hash_step(uint64_t h, int64_t time_ns, uint64_t word1)
{
    h = (h ^ (uint64_t)time_ns) * HS_HASH_MUL;
    h = (h ^ word1) * HS_HASH_MUL;
    return h;
}

#endif /* HS_SAMPLER_H */
