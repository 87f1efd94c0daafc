/* hs_engine.cu -- C-ABI of the H100 discrete-event engine (include/hs_b200.h).
 *
 * Host side of the boundary: validates and uploads the flat model, owns the
 * device buffers (replica state, queue rings, per-replica outputs), picks the
 * kernel (lane engine for the single-server topology, warp engine otherwise),
 * launches on the engine's CUDA stream and times the launches with CUDA events
 * recorded on that same stream.  No torch types, no CPU fallback.
 */
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/hs_b200.h"
#include "hs_lane_engine.cuh"
#include "hs_warp_engine.cuh"
#include "hs_thread_engine.cuh"
#include "hs_totals.cuh"
#include "hs_sketch.h"

static thread_local char g_err[512] = "";

static int fail(int code, const char *fmt, ...)
{
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return code;
}

#define CUDA_TRY(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e_ = (expr);                                                                \
        if (e_ != cudaSuccess)                                                                  \
            return fail(HS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_),    \
                        __FILE__, __LINE__);                                                    \
    } while (0)

struct dev_buf {
    void *p = nullptr; size_t n = 0;
    int ensure(size_t bytes) {
        if (bytes <= n && p) return 0;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        if (bytes == 0) return 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e != cudaSuccess) return fail(HS_ERR_CUDA, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        n = bytes;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

struct hs_engine {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    uint64_t launches = 0;
    hs_launch_info last_launch = {};                /* engine == 0: nothing launched yet */
    int sm_count = 132;

    /* model (host copy + device copy) */
    bool have_model = false;
    std::vector<hs_entity_desc> ents;
    std::vector<int32_t> backends, key_table;
    std::vector<double> cell_d0; std::vector<int32_t> cell_i0;
    std::vector<hs_profile_desc> profiles;      /* STEP rows: p[2] = device address of the row's table */
    std::vector<hs_profile_desc> profiles_raw;  /* as uploaded, p[2] of STEP rows zeroed (for the same-model test) */
    std::vector<double> profile_table;
    uint32_t n_cells = 0;
    dev_buf d_ents, d_backends, d_key_table, d_cell_d0, d_cell_i0, d_profiles, d_profile_table, d_sketch_tab, d_key_cdf;
    std::vector<int32_t> sketch_tab;
    std::vector<double> key_cdf;
    std::vector<uint64_t> sk_off, sk_moff;      /* hs_sketch_layout of the model */
    uint64_t sk_total = 0, sk_mtotal = 0;
    dev_buf d_sketch, d_sketch_merged;
    bool lane_ok = false;
    hs_lane_model lane_model;

    /* last run */
    bool have_run = false;
    hs_run_params last;
    int last_engine = 0;
    uint32_t last_ring = 0;
    dev_buf d_conts, d_hist, d_cell_totals; bool hist_on = false;
    dev_buf d_trace_arr, d_trace_svc; uint64_t n_trace_arr = 0, n_trace_svc = 0; uint32_t trace_replicas = 0;
    dev_buf d_state, d_rings, d_summ, d_stats, d_rec, d_smp, d_svc, d_partials, d_totals, d_srv_index, d_counter;
    /* linked partitions */
    uint32_t outbox_cap = 0, inbox_cap = 0;
    std::vector<int32_t> srv_index_host;        /* what d_srv_index holds */
    dev_buf d_outbox, d_outbox_n, d_inbox, d_inbox_n;
    uint32_t link_replicas = 0;                 /* replicas the outbox / inbox buffers are sized for */
};

/* ---- validation ----------------------------------------------------------- */

static int validate_model(const hs_model_desc *m)
{
    if (!m) return fail(HS_ERR_INVALID, "model is NULL");
    if (m->abi_version != HS_ABI_VERSION) return fail(HS_ERR_INVALID, "abi_version %u != %u", m->abi_version, HS_ABI_VERSION);
    if (m->n_entities == 0 || m->n_entities > 65535 || !m->entities) return fail(HS_ERR_INVALID, "n_entities must be 1..65535");
    uint32_t n = m->n_entities;
    int n_src = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const hs_entity_desc &e = m->entities[i];
        switch (e.kind) {
        case HS_ENT_SOURCE:
            n_src++;
            if (e.target < 0 || (uint32_t)e.target >= n) return fail(HS_ERR_INVALID, "entity %u: source target %d out of range", i, e.target);
            if (m->entities[e.target].kind == HS_ENT_REMOTE) return fail(HS_ERR_INVALID, "entity %u: a source's target must be in its own partition (parallel/validation.py:53-71)", i);
            if (m->entities[e.target].kind == HS_ENT_SOURCE) return fail(HS_ERR_INVALID, "entity %u: source targets a source", i);
            if (e.i3 < 0 || (uint32_t)e.i3 > m->n_profiles) return fail(HS_ERR_INVALID, "entity %u: profile index %d out of range", i, e.i3);
            if (e.i3 > 0 && !m->profiles) return fail(HS_ERR_INVALID, "profiles is NULL");
            if (e.i3 > 0 && (m->profiles[e.i3 - 1].kind < HS_PROF_CONSTANT || m->profiles[e.i3 - 1].kind > HS_PROF_STEP))
                return fail(HS_ERR_INVALID, "entity %u: unknown profile kind", i);
            if (e.i3 > 0 && m->profiles[e.i3 - 1].kind == HS_PROF_LINEAR_RAMP && !(m->profiles[e.i3 - 1].p[0] > 0.0))
                return fail(HS_ERR_INVALID, "entity %u: LinearRampProfile duration must be > 0", i);
            if (e.i3 > 0) {     /* a rate that reaches zero sends the reference's bracket search to times beyond int64 ns */
                const hs_profile_desc &pr = m->profiles[e.i3 - 1];
                bool ok = pr.kind == HS_PROF_LINEAR_RAMP ? (pr.p[1] > 0.0 && pr.p[2] > 0.0)
                        : pr.kind == HS_PROF_SPIKE ? (pr.p[0] > 0.0 && pr.p[1] > 0.0 && pr.p[2] >= 0.0 && pr.p[3] >= 0.0)
                        : pr.kind == HS_PROF_STEP ? true : (pr.p[0] > 0.0);
                if (pr.kind == HS_PROF_STEP) {
                    const double off = pr.p[0], nb = pr.p[1];
                    if (!(off >= 0.0 && nb >= 0.0 && nb <= 65536.0) || !m->profile_table ||
                        (uint64_t)off + 2 * (uint64_t)nb + 1 > m->n_profile_table)
                        return fail(HS_ERR_INVALID, "entity %u: step profile table out of range", i);
                    const double *tab = m->profile_table + (uint64_t)off;
                    const uint64_t nbi = (uint64_t)nb;
                    for (uint64_t k = 0; k + 1 < nbi; ++k) if (!(tab[k] < tab[k + 1])) return fail(HS_ERR_INVALID, "entity %u: step profile breakpoints must ascend", i);
                    for (uint64_t k = 0; k <= nbi; ++k) ok = ok && tab[nbi + k] > 0.0;
                }
                if (!ok) return fail(HS_ERR_INVALID, "entity %u: profile rates must stay > 0", i);
            }
            if (e.i3 == 0 && !(e.d0 > 0.0)) return fail(HS_ERR_INVALID, "entity %u: source rate must be > 0 (arrival_time_provider.py:75)", i);
            if (e.i0 != HS_ARR_CONSTANT && e.i0 != HS_ARR_POISSON) return fail(HS_ERR_INVALID, "entity %u: bad arrival kind", i);
            if (e.i2 < 0 || (e.i2 > 0 && (e.i1 <= 0 || !m->key_cdf || (uint64_t)(e.i2 - 1) + (uint64_t)e.i1 > m->n_key_cdf)))
                return fail(HS_ERR_INVALID, "entity %u: Zipf key table out of range", i);
            if (e.i2 > 0) {
                const double *c = m->key_cdf + (e.i2 - 1);
                for (int32_t k = 0; k < e.i1; ++k)
                    if (!(c[k] >= 0.0 && c[k] <= 1.0) || (k > 0 && c[k] < c[k - 1])) return fail(HS_ERR_INVALID, "entity %u: cumulative key probabilities must be non-decreasing in [0, 1]", i);
            }
            if (e.i1 < 0 || (e.i1 > 0 && m->key_population > 0 && (uint32_t)e.i1 != m->key_population)) return fail(HS_ERR_INVALID, "entity %u: key population %d != key_table length %u", i, e.i1, m->key_population);
            break;
        case HS_ENT_SERVER:
            if (e.target >= (int32_t)n) return fail(HS_ERR_INVALID, "entity %u: downstream out of range", i);
            if (e.target >= 0 && m->entities[e.target].kind == HS_ENT_SOURCE) return fail(HS_ERR_INVALID, "entity %u: downstream is a source", i);
            if (e.i0 < 1) return fail(HS_ERR_INVALID, "entity %u: max_concurrent must be >= 1, got %d (concurrency.py:86)", i, e.i0);
            if (e.i1 != HS_Q_FIFO && e.i1 != HS_Q_LIFO) return fail(HS_ERR_INVALID, "entity %u: bad queue policy", i);
            if (e.i2 != HS_SVC_CONSTANT && e.i2 != HS_SVC_EXPONENTIAL) return fail(HS_ERR_INVALID, "entity %u: bad service kind", i);
            if (e.i2 == HS_SVC_EXPONENTIAL && !(e.d0 > 0.0)) return fail(HS_ERR_INVALID, "entity %u: exponential mean must be > 0", i);
            if (e.d0 < 0.0) return fail(HS_ERR_INVALID, "entity %u: negative service time", i);
            break;
        case HS_ENT_CACHE_SERVER:
            if (e.target != -1) return fail(HS_ERR_INVALID, "entity %u: a CachingServer forwards nothing (its generator returns [])", i);
            if (e.i0 < 1 || e.i0 > (1 << 20)) return fail(HS_ERR_INVALID, "entity %u: key slots must be in [1, 2^20]", i);
            if (e.i1 != HS_Q_FIFO && e.i1 != HS_Q_LIFO) return fail(HS_ERR_INVALID, "entity %u: bad queue policy", i);
            if (e.i2 < 0 || e.i3 < 0 || e.l0 < 0) return fail(HS_ERR_INVALID, "entity %u: negative latency", i);
            if (!(e.d0 > 0.0)) return fail(HS_ERR_INVALID, "entity %u: ttl must be > 0 (eviction_policies.py:174)", i);
            break;
        case HS_ENT_SINK: case HS_ENT_COUNTER: break;
        case HS_ENT_REMOTE:
            if (e.i0 < 0 || e.i0 >= 16 || e.i1 < 0) return fail(HS_ERR_INVALID, "entity %u: REMOTE row needs a link slot in 0..15 and a destination entity id", i);
            if (m->outbox_cap == 0) return fail(HS_ERR_INVALID, "entity %u: a model with REMOTE rows needs outbox_cap > 0", i);
            break;
        case HS_ENT_SKETCH: {
            if (e.i0 < HS_SK_HLL || e.i0 > HS_SK_RESERVOIR) return fail(HS_ERR_INVALID, "entity %u: unknown sketch algorithm %d", i, e.i0);
            if (e.l0 < 0 || e.l0 > INT32_MAX) return fail(HS_ERR_INVALID, "entity %u: sketch key population must be >= 0", i);
            if (e.l0 == 0 && (e.i0 == HS_SK_HLL || e.i0 == HS_SK_CMS || e.i0 == HS_SK_BLOOM)) {    /* hashed on the device */
                const uint64_t words = e.i0 == HS_SK_CMS ? 2u * (uint64_t)e.i2 : 2u;
                if (e.i0 == HS_SK_HLL && (e.i2 < 4 || e.i2 > 16)) return fail(HS_ERR_INVALID, "entity %u: precision must be in [4, 16], got %d (hyperloglog.py:101)", i, e.i2);
                if (e.i0 != HS_SK_HLL && (e.i2 < 1 || e.i3 < 1)) return fail(HS_ERR_INVALID, "entity %u: sketch dimensions must be >= 1", i);
                if (e.i1 < 0 || !m->sketch_tables || (uint64_t)e.i1 + words > m->n_sketch_table)
                    return fail(HS_ERR_INVALID, "entity %u: sketch seed words out of range", i);
                break;
            }
            if (e.i0 == HS_SK_RESERVOIR) {
                if (e.i2 < 1) return fail(HS_ERR_INVALID, "entity %u: size must be positive (reservoir.py:68)", i);
                if (e.i1 < 0 || !m->sketch_tables || (uint64_t)e.i1 + 625u > m->n_sketch_table)
                    return fail(HS_ERR_INVALID, "entity %u: generator state (625 words) out of range", i);
                if ((uint32_t)m->sketch_tables[e.i1 + 624] > 624u) return fail(HS_ERR_INVALID, "entity %u: generator index must be <= 624", i);
                break;
            }
            if (e.l0 == 0 && e.i0 == HS_SK_TOPK) { if (e.i2 < 1) return fail(HS_ERR_INVALID, "entity %u: k must be positive (topk.py:79)", i); break; }
            if (e.l0 == 0 && e.i0 != HS_SK_TDIGEST) return fail(HS_ERR_INVALID, "entity %u: sketch key population must be >= 1", i);
            if (e.i0 == HS_SK_HLL && (e.i2 < 4 || e.i2 > 16)) return fail(HS_ERR_INVALID, "entity %u: precision must be in [4, 16], got %d (hyperloglog.py:101)", i, e.i2);
            if (e.i0 == HS_SK_CMS && (e.i2 < 1 || e.i3 < 1)) return fail(HS_ERR_INVALID, "entity %u: width and depth must be >= 1 (count_min_sketch.py:88-91)", i);
            if (e.i0 == HS_SK_BLOOM && (e.i2 < 1 || e.i3 < 1)) return fail(HS_ERR_INVALID, "entity %u: size_bits and num_hashes must be >= 1 (bloom_filter.py:101-104)", i);
            if (e.i0 == HS_SK_TOPK && e.i2 < 1) return fail(HS_ERR_INVALID, "entity %u: k must be positive (topk.py:79)", i);
            if (e.i0 == HS_SK_TDIGEST) {
                if (!(e.d0 > 0.0)) return fail(HS_ERR_INVALID, "entity %u: compression must be positive (tdigest.py:79)", i);
                if (e.i2 < 1 || e.i2 != (int32_t)(e.d0 * 2.0)) return fail(HS_ERR_INVALID, "entity %u: buffer size must be int(compression * 2) >= 1 (tdigest.py:88)", i);
                if (e.i3 < 2 * e.i2) return fail(HS_ERR_INVALID, "entity %u: centroid capacity must be >= 2 x buffer size", i);
                break;
            }
            const uint64_t rows = e.i0 == HS_SK_HLL ? 2u : e.i0 == HS_SK_TOPK ? 0u : (uint64_t)e.i2;
            if (rows && (e.i1 < 0 || !m->sketch_tables || (uint64_t)e.i1 + rows * (uint64_t)e.l0 > m->n_sketch_table))
                return fail(HS_ERR_INVALID, "entity %u: sketch table out of range", i);
            const int32_t *tab = rows ? m->sketch_tables + e.i1 : nullptr;
            for (int64_t k = 0; rows && k < e.l0; ++k) {
                if (e.i0 == HS_SK_HLL) {
                    if (tab[k] < 0 || tab[k] >= (1 << e.i2) || tab[e.l0 + k] < 1 || tab[e.l0 + k] > 64 - e.i2 + 1)
                        return fail(HS_ERR_INVALID, "entity %u: HLL table entry %lld out of range", i, (long long)k);
                } else {
                    for (int32_t row = 0; row < e.i2; ++row)
                        if (tab[(int64_t)row * e.l0 + k] < 0 || tab[(int64_t)row * e.l0 + k] >= e.i3)
                            return fail(HS_ERR_INVALID, "entity %u: %s of key %lld out of range", i, e.i0 == HS_SK_CMS ? "CMS column" : "Bloom bit", (long long)k);
                }
            }
            for (uint32_t j = 0; j < n; ++j)
                if (m->entities[j].kind == HS_ENT_SOURCE && m->entities[j].i1 > e.l0)
                    return fail(HS_ERR_INVALID, "entity %u: a source draws keys from %d values, the sketch table covers %lld", i, m->entities[j].i1, (long long)e.l0);
            break;
        }
        case HS_ENT_PROBE: {
            if (e.target < 0 || (uint32_t)e.target >= n) return fail(HS_ERR_INVALID, "entity %u: probe target out of range", i);
            const int tk = m->entities[e.target].kind;
            const bool ok = (e.i0 >= HS_METRIC_DEPTH && e.i0 <= HS_METRIC_STATS_DROPPED) ? tk == HS_ENT_SERVER
                          : e.i0 == HS_METRIC_EVENTS_RECEIVED ? tk == HS_ENT_SINK
                          : e.i0 == HS_METRIC_TOTAL ? tk == HS_ENT_COUNTER
                          : e.i0 == HS_METRIC_GENERATED_COUNT ? tk == HS_ENT_SOURCE : false;
            if (!ok) return fail(HS_ERR_INVALID, "entity %u: metric %d is not defined for the probed entity", i, e.i0);
            break;
        }
        case HS_ENT_LB:
            if (e.i0 != HS_LB_ROUND_ROBIN && e.i0 != HS_LB_KEY_TABLE) return fail(HS_ERR_INVALID, "entity %u: bad LB strategy", i);
            if (e.i2 < 0 || e.i1 < 0 || (uint32_t)(e.i1 + e.i2) > m->n_backends) return fail(HS_ERR_INVALID, "entity %u: backend list out of range", i);
            if (e.i2 > 0 && !m->backends) return fail(HS_ERR_INVALID, "backends is NULL");
            for (int b = 0; b < e.i2; ++b) {
                int be = m->backends[e.i1 + b];
                if (be < 0 || (uint32_t)be >= n) return fail(HS_ERR_INVALID, "entity %u: backend %d out of range", i, be);
                int bk = m->entities[be].kind;
                if (bk != HS_ENT_SERVER && bk != HS_ENT_CACHE_SERVER && bk != HS_ENT_SINK && bk != HS_ENT_COUNTER) return fail(HS_ERR_INVALID, "entity %u: backend %d must be a Server, CachingServer, Sink or Counter", i, be);
            }
            if (e.i0 == HS_LB_KEY_TABLE) {
                if (!m->key_table || m->key_population == 0) return fail(HS_ERR_INVALID, "entity %u: key table missing", i);
                for (uint32_t k = 0; k < m->key_population; ++k)
                    if (m->key_table[k] < 0 || m->key_table[k] >= e.i2) return fail(HS_ERR_INVALID, "key_table[%u] = %d out of range", k, m->key_table[k]);
            }
            break;
        default: return fail(HS_ERR_INVALID, "entity %u: unknown kind %d", i, e.kind);
        }
    }
    if (m->n_cells && (!m->cell_d0 || !m->cell_i0)) return fail(HS_ERR_INVALID, "cells without tables");
    for (uint32_t c = 0; c < m->n_cells; ++c)
        for (uint32_t i = 0; i < n; ++i) {
            const hs_entity_desc &e = m->entities[i];
            double d = m->cell_d0[(size_t)c * n + i]; int32_t v = m->cell_i0[(size_t)c * n + i];
            if (e.kind == HS_ENT_SOURCE && e.i3 == 0 && !(d > 0.0)) return fail(HS_ERR_INVALID, "cell %u: source rate must be > 0", c);
            if (e.kind == HS_ENT_SERVER && (v < 1 || d < 0.0)) return fail(HS_ERR_INVALID, "cell %u: bad server override", c);
            if (e.kind != HS_ENT_SERVER && v != e.i0) return fail(HS_ERR_INVALID, "cell %u: i0 override only applies to servers", c);
        }
    return HS_OK;
}

/* a server's concurrency limit, maximised over the sweep cells */
static int32_t max_concurrency(const hs_engine *E, uint32_t i)
{
    const size_t n = E->ents.size();
    int32_t c = E->ents[i].i0;
    for (uint32_t k = 0; k < E->n_cells; ++k) c = std::max(c, E->cell_i0[(size_t)k * n + i]);
    return c;
}

/* Lane engine eligibility: exactly Source -> Server(concurrency <= 64) -> Sink|Counter|none, and not a partition of a
 * linked run (the lane kernel has no outbox and no inbox). */
static bool classify_lane(hs_engine *E)
{
    const auto &en = E->ents;
    size_t n = en.size();
    if (n < 2 || n > 3 || E->outbox_cap || E->inbox_cap) return false;
    int src = -1, srv = -1, dst = -1;
    for (size_t i = 0; i < n; ++i) {
        if (en[i].kind == HS_ENT_SOURCE) { if (src >= 0) return false; src = (int)i; }
        else if (en[i].kind == HS_ENT_SERVER) { if (srv >= 0) return false; srv = (int)i; }
        else if (en[i].kind == HS_ENT_SINK || en[i].kind == HS_ENT_COUNTER) { if (dst >= 0) return false; dst = (int)i; }
        else return false;
    }
    if (src < 0 || srv < 0) return false;
    if (en[src].target != srv || en[src].i1 != 0) return false;
    if (en[srv].target != dst) { if (!(en[srv].target < 0 && dst < 0)) return false; }
    const int32_t c_max = max_concurrency(E, (uint32_t)srv);
    if (c_max > 64) return false;
    hs_lane_model &L = E->lane_model;
    memset(&L, 0, sizeof L);
    L.src_id = src; L.srv_id = srv; L.dst_id = en[srv].target;
    L.dst_kind = L.dst_id >= 0 ? en[L.dst_id].kind : 0;
    L.arr_kind = en[src].i0; L.svc_kind = en[srv].i2; L.policy = en[srv].i1; L.n_entities = (int32_t)n;
    L.capacity = en[srv].l0; L.stop_after = en[src].l0;
    L.rate = en[src].d0; L.mean = en[srv].d0;
    L.concurrency = en[srv].i0; L.c_max = c_max;
    L.cell_i0 = (const int32_t *)E->d_cell_i0.p;
    L.has_profile = en[src].i3 > 0;
    if (L.has_profile) L.prof = E->profiles[en[src].i3 - 1];
    L.n_cells = E->n_cells;
    L.cell_d0 = (const double *)E->d_cell_d0.p;
    return true;
}

static uint32_t pow2_at_least(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }

/* ---- one launcher per kernel ----------------------------------------------- */

/* The launch between the run's two timing events: hs_last_run_ms brackets the kernel alone, so every other piece of
 * host work (function attributes, uploads, memsets) is issued before this call.  `info` is the launch's geometry
 * (grid, block, smem) and what hs_last_launch reports of it. */
template <typename Kernel, typename... Args>
static int timed_launch(hs_engine *E, const hs_launch_info &info, Kernel kern, Args... args)
{
    CUDA_TRY(cudaEventRecord(E->ev0, E->stream));
    kern<<<info.grid, info.block, info.smem, E->stream>>>(args...);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(E->ev1, E->stream));
    E->launches += 1;
    E->last_launch = info;
    return HS_OK;
}

#define HS_K4(K, F) K<F>, K<F + 1>, K<F + 2>, K<F + 3>

static int launch_lane(hs_engine *E, const hs_kernel_run &R, const hs_kernel_out &O, bool want_hash, bool want_rec)
{
    const hs_lane_model &M = E->lane_model;
    const uint32_t n = R.n_replicas;
    int rc;
    if ((rc = E->d_state.ensure((size_t)n * sizeof(hs_lane_state)))) return rc;
    if ((rc = E->d_rings.ensure((size_t)n * R.ring * sizeof(hs_ring_entry)))) return rc;
    if ((rc = E->d_conts.ensure(std::max<size_t>(64, (size_t)n * M.c_max * sizeof(hs_cont))))) return rc;
    const bool simple = !M.has_profile && !R.trace_arr && !R.trace_svc && M.arr_kind == HS_ARR_POISSON &&
                        M.svc_kind == HS_SVC_EXPONENTIAL && M.policy == HS_Q_FIFO && M.capacity < 0 &&
                        M.stop_after < 0 && M.dst_id >= 0 && M.dst_kind == HS_ENT_SINK && M.c_max == 1;
    const int fl = (want_hash ? HS_LF_HASH : 0) | (want_rec ? HS_LF_REC : 0) |
                   (M.has_profile ? HS_LF_PROFILE : 0) | (simple ? HS_LF_SIMPLE : 0);
    using kernel = void (*)(hs_lane_model, hs_kernel_run, hs_lane_state *, hs_ring_entry *, hs_cont *, hs_kernel_out);
    static const kernel kernels[] = {HS_K4(hs_lane_kernel, 0), HS_K4(hs_lane_kernel, 4),     /* fl <= 11: the SIMPLE */
                                     HS_K4(hs_lane_kernel, 8)};                               /* model has no profile */
    const hs_launch_info info = {2, HS_KERNEL_LANE, (uint32_t)fl, 1, 0, (n + HS_LANE_THREADS - 1) / HS_LANE_THREADS,
                                 HS_LANE_THREADS, 0};
    return timed_launch(E, info, kernels[fl], M, R, (hs_lane_state *)E->d_state.p, (hs_ring_entry *)E->d_rings.p,
                        (hs_cont *)E->d_conts.p, O);
}

static const uint32_t HS_WARP_SMEM_MAX = 227 * 1024 - 1024;      /* dynamic shared memory of a warp-engine CTA */

/* What the warp and the thread engine share: the future-event slots, the servers' queue-ring indices, the replica
 * state and queue-ring buffers, and the model flags (*fl). */
static int general_setup(hs_engine *E, const hs_kernel_run &R, bool thread, bool want_hash, bool want_rec,
                         hs_warp_model &M, int *fl)
{
    const uint32_t n = R.n_replicas;
    const uint32_t ne = (uint32_t)E->ents.size();
    /* FEL slots: one pending SourceEvent per source, one ProcessContinuation per busy
     * server slot, plus the same-timestamp protocol events in flight. */
    uint64_t live = 24;
    uint32_t n_servers = 0;
    bool any_profile = false;
    std::vector<int32_t> srv_index(ne, -1);
    for (uint32_t i = 0; i < ne; ++i) {
        const hs_entity_desc &e = E->ents[i];
        if (e.kind == HS_ENT_SOURCE) { live += 2; any_profile = any_profile || e.i3 > 0; }
        if (e.kind == HS_ENT_SERVER) live += (uint64_t)max_concurrency(E, i) + 1;
        if (e.kind == HS_ENT_CACHE_SERVER) live += 64;      /* no concurrency limit: one pending continuation per request in service;
                                                              64 covers 10 000 requests/s through the ~6 ms of a miss (overflow is flagged) */
        if (e.kind == HS_ENT_SERVER || e.kind == HS_ENT_CACHE_SERVER) srv_index[i] = (int32_t)n_servers++;
    }
    live += E->inbox_cap;                            /* what a barrier can deliver is scheduled at once */
    const uint32_t S = (uint32_t)((live + 31) / 32) * 32;
    if (S > 65535) return fail(HS_ERR_INVALID, "model needs %u future-event slots (limit 65535)", S);
    /* thread engine: 4-ary key heap + payload slots instead of the warp engine's SoA slot table */
    const uint32_t block_bytes = thread
        ? hs_thread_offsets(ne, S).total
        : (uint32_t)(sizeof(hs_warp_hdr) + (size_t)ne * sizeof(hs_went) + (((size_t)S * 46 + 15) / 16) * 16 +
                     (size_t)HS_W_NCAP * sizeof(hs_wnow));
    /* the warp engine stages a replica's block (and an mbarrier slot) in shared memory */
    if (!thread && 16 + block_bytes > HS_WARP_SMEM_MAX)
        return fail(HS_ERR_INVALID, "model too large for the warp engine (%u B of state per replica)", 16 + block_bytes);
    int rc;
    if ((rc = E->d_state.ensure((size_t)n * block_bytes))) return rc;
    if ((rc = E->d_rings.ensure(std::max<size_t>(16, (size_t)n * n_servers * R.ring * sizeof(hs_wring_entry))))) return rc;
    if ((rc = E->d_srv_index.ensure(ne * 4 + 16))) return rc;
    if (E->srv_index_host != srv_index) {            /* uploaded once per model: the window loop of a linked run stays asynchronous */
        E->srv_index_host = srv_index;
        CUDA_TRY(cudaMemcpyAsync(E->d_srv_index.p, E->srv_index_host.data(), ne * 4, cudaMemcpyHostToDevice, E->stream));
        CUDA_TRY(cudaStreamSynchronize(E->stream));
    }
    M.ents = (const hs_entity_desc *)E->d_ents.p;
    M.backends = (const int32_t *)E->d_backends.p; M.key_table = (const int32_t *)E->d_key_table.p;
    M.srv_index = (const int32_t *)E->d_srv_index.p;
    M.cell_d0 = (const double *)E->d_cell_d0.p; M.cell_i0 = (const int32_t *)E->d_cell_i0.p;
    M.profiles = (const hs_profile_desc *)E->d_profiles.p;
    M.sketch_tables = (const int32_t *)E->d_sketch_tab.p; M.sk_total = E->sk_total;
    M.key_cdf = (const double *)E->d_key_cdf.p;
    M.n_entities = ne; M.n_cells = E->n_cells; M.n_servers = n_servers; M.fel_slots = S; M.block_bytes = block_bytes;
    M.n_backends = (uint32_t)E->backends.size(); M.model_bytes = 0;
    M.outbox_cap = E->outbox_cap; M.inbox_cap = E->inbox_cap;
    M.fixed_slots = 0; M.pad_ = 0;
    *fl = (want_hash ? HS_WF_HASH : 0) | (want_rec ? HS_WF_REC : 0) | (any_profile ? HS_WF_PROFILE : 0);
    return HS_OK;
}

static int launch_warp(hs_engine *E, const hs_kernel_run &R, const hs_kernel_out &O, bool want_hash, bool want_rec)
{
    hs_warp_model M;
    int fl, rc;
    if ((rc = general_setup(E, R, false, want_hash, want_rec, M, &fl))) return rc;
    /* per warp its replica's block behind an mbarrier slot; per CTA a copy of the model tables when they fit */
    const uint32_t ne = M.n_entities;
    const uint32_t per_warp = 16 + M.block_bytes;
    M.model_bytes = (uint32_t)((ne * sizeof(hs_entity_desc) + ne * 4 + E->backends.size() * 4 + 15) / 16 * 16);
    if (per_warp + M.model_bytes > HS_WARP_SMEM_MAX) M.model_bytes = 0;      /* tables stay in global memory */
    const uint32_t smem_budget = 200 * 1024;
    uint32_t warps = std::min<uint32_t>(8, std::max<uint32_t>(1, (smem_budget / 2) / per_warp));
    while (warps > 1 && per_warp * warps + M.model_bytes > HS_WARP_SMEM_MAX) warps--;
    const uint32_t smem = per_warp * warps + M.model_bytes;
    uint32_t blocks_per_sm = std::max<uint32_t>(1, std::min<uint32_t>((227 * 1024) / (smem + 1024), 64 / warps));
    if (blocks_per_sm * warps * 32 > 2048) blocks_per_sm = 2048 / (warps * 32);
    const uint32_t grid = std::min<uint32_t>((R.n_replicas + warps - 1) / warps, (uint32_t)E->sm_count * blocks_per_sm);
    if ((rc = E->d_counter.ensure(16))) return rc;
    CUDA_TRY(cudaMemsetAsync(E->d_counter.p, 0, 16, E->stream));
    using kernel = void (*)(hs_warp_model, hs_kernel_run, unsigned char *, hs_wring_entry *, hs_kernel_out, unsigned int *);
    static const kernel kernels[] = {HS_K4(hs_warp_kernel, 0), HS_K4(hs_warp_kernel, 4)};
    CUDA_TRY(cudaFuncSetAttribute(kernels[fl], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const hs_launch_info info = {1, HS_KERNEL_WARP, (uint32_t)fl, 1, 0, grid, warps * 32, smem};
    return timed_launch(E, info, kernels[fl], M, R, (unsigned char *)E->d_state.p,
                        (hs_wring_entry *)E->d_rings.p, O, (unsigned int *)E->d_counter.p);
}

static int launch_thread(hs_engine *E, hs_kernel_run R, const hs_kernel_out &O, bool want_hash, bool want_rec, bool linked)
{
    hs_warp_model M;
    int fl, rc;
    if ((rc = general_setup(E, R, true, want_hash, want_rec, M, &fl))) return rc;
    const uint32_t n = R.n_replicas, ne = M.n_entities, S = M.fel_slots;
    /* entity-owned payload slots: every entity has at most one pending future event; delivered events need slots of their own */
    bool fixed = ne <= S && E->inbox_cap == 0;
    for (uint32_t i = 0; i < ne && fixed; ++i) {
        const int32_t kind = E->ents[i].kind;
        if (kind == HS_ENT_CACHE_SERVER || (kind == HS_ENT_SERVER && max_concurrency(E, i) != 1)) fixed = false;
    }
    M.fixed_slots = fixed ? 1u : 0u;
    /* replicas per warp: enough warps to fill the register file (16 warps of 128 registers per SM),
     * and no more lanes per warp than that needs -- a warp's iteration costs the sum of the distinct
     * paths its lanes take. */
    const uint32_t rpw = std::min<uint32_t>(32, pow2_at_least((uint32_t)((n + (uint64_t)E->sm_count * 16 - 1) / ((uint64_t)E->sm_count * 16))));
    R.lane_stride = 32 / rpw;
    const uint32_t tblocks = (uint32_t)(((uint64_t)n * R.lane_stride + HS_THREAD_BLOCK - 1) / HS_THREAD_BLOCK);
    /* shared memory of a block: the now tier (HS_T_KS entries x 48 B per replica column) and, next to it, whole top
     * levels of the key heap: at most three (1 + 4 + 16 keys) and at most 20 KB per block together.  Shared memory is
     * carved out of the L1 the replicas' state lives in, and deep levels are read at scattered indices (bank
     * conflicts): on the 64-server farm at 8 replicas per warp, 5 / 21 / 85 keys per replica in shared memory ran at
     * 8.99e9 / 9.25e9 / 8.71e9 events/s. */
    const uint32_t rpb = HS_THREAD_BLOCK / R.lane_stride;
    const uint32_t budget = std::min<uint32_t>(21u, (20480u / 16u - HS_T_KS * 3u * rpb) / rpb);          /* keys per replica */
    uint32_t top = 0, level = 1, total = 0;
    while (total + level <= budget && total + level <= S) { total += level; level *= HS_T_ARITY; top = total; }
    R.heap_top = (top < 1 + HS_T_ARITY || R.lane_stride == 32) ? 0 : top;  /* one replica per warp: its heap sits in L1 anyway */
    const size_t dyn_smem = (size_t)(HS_T_KS * 3u + R.heap_top) * rpb * 16;
    using kernel = void (*)(hs_warp_model, hs_kernel_run, unsigned char *, hs_wring_entry *, hs_kernel_out);
    static const kernel kernels[] = {HS_K4(hs_thread_kernel, 0), HS_K4(hs_thread_kernel, 4), HS_K4(hs_thread_kernel, 8),
                                     HS_K4(hs_thread_kernel, 12), HS_K4(hs_thread_kernel, 16), HS_K4(hs_thread_kernel, 20),
                                     HS_K4(hs_thread_kernel, 24), HS_K4(hs_thread_kernel, 28)};
    static const kernel wide_kernels[] = {HS_K4(hs_thread_kernel_wide, 0), HS_K4(hs_thread_kernel_wide, 4)};
    /* small launches (every block resident at 4 blocks per SM, no shared-memory heap top, not linked): the spill-free
     * instantiation, see hs_thread_kernel_wide */
    const bool wide = !R.heap_top && !linked && tblocks <= (uint32_t)E->sm_count * HS_T_WIDE_BLOCKS;
    if (!wide) fl |= (R.heap_top ? HS_WF_HEAPTOP : 0) | (linked ? HS_WF_LINKED : 0);
    const hs_launch_info info = {3, wide ? (uint32_t)HS_KERNEL_THREAD_WIDE : (uint32_t)HS_KERNEL_THREAD, (uint32_t)fl,
                                 R.lane_stride, R.heap_top, tblocks, HS_THREAD_BLOCK, (uint32_t)dyn_smem};
    return timed_launch(E, info, wide ? wide_kernels[fl] : kernels[fl], M, R, (unsigned char *)E->d_state.p,
                        (hs_wring_entry *)E->d_rings.p, O);
}
#undef HS_K4

/* ---- entry points ------------------------------------------------------- */

extern "C" {

uint32_t hs_version(void) { return HS_ABI_VERSION; }

int hs_last_error(char *buf, int len)
{
    int n = (int)strlen(g_err);
    if (buf && len > 0) { strncpy(buf, g_err, (size_t)len - 1); buf[len - 1] = 0; }
    return n;
}

int hs_model_validate(const hs_model_desc *model) { return validate_model(model); }

int hs_engine_create(int device, void *stream, hs_engine **out)
{
    if (!out) return fail(HS_ERR_INVALID, "out is NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(HS_ERR_NO_DEVICE, "no CUDA device (%s); the engine has no CPU path", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
    if (device < 0 || device >= count) return fail(HS_ERR_INVALID, "device %d out of range (0..%d)", device, count - 1);
    CUDA_TRY(cudaSetDevice(device));
    hs_engine *E = new hs_engine();
    E->device = device;
    if (stream) { E->stream = (cudaStream_t)stream; E->own_stream = false; }
    else { CUDA_TRY(cudaStreamCreateWithFlags(&E->stream, cudaStreamNonBlocking)); E->own_stream = true; }
    CUDA_TRY(cudaEventCreate(&E->ev0));
    CUDA_TRY(cudaEventCreate(&E->ev1));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    E->sm_count = prop.multiProcessorCount;
    *out = E;
    return HS_OK;
}

int hs_engine_destroy(hs_engine *E)
{
    if (!E) return HS_OK;
    cudaSetDevice(E->device);
    cudaStreamSynchronize(E->stream);
    dev_buf *bufs[] = {&E->d_ents, &E->d_backends, &E->d_key_table, &E->d_cell_d0, &E->d_cell_i0, &E->d_state,
                       &E->d_rings, &E->d_summ, &E->d_stats, &E->d_rec, &E->d_smp, &E->d_svc, &E->d_partials, &E->d_totals,
                       &E->d_srv_index, &E->d_counter, &E->d_trace_arr, &E->d_trace_svc, &E->d_profiles, &E->d_profile_table, &E->d_hist, &E->d_cell_totals, &E->d_conts,
                       &E->d_sketch_tab, &E->d_sketch, &E->d_sketch_merged, &E->d_key_cdf,
                       &E->d_outbox, &E->d_outbox_n, &E->d_inbox, &E->d_inbox_n};
    for (dev_buf *b : bufs) b->release();
    if (E->ev0) cudaEventDestroy(E->ev0);
    if (E->ev1) cudaEventDestroy(E->ev1);
    if (E->own_stream && E->stream) cudaStreamDestroy(E->stream);
    delete E;
    return HS_OK;
}

int hs_model_upload(hs_engine *E, const hs_model_desc *m)
{
    if (!E) return fail(HS_ERR_INVALID, "engine is NULL");
    int rc = validate_model(m);
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(E->device));
    uint32_t n = m->n_entities;
    /* Re-uploading the model that is already resident (byte-identical tables) keeps a paused run resumable:
     * a caller that sends its model with every window, as Simulation.run_ensemble does, still continues
     * the same run.  Any difference starts over. */
    auto same_bytes = [](const void *a, size_t na, const void *b, size_t nb) { return na == nb && (na == 0 || memcmp(a, b, na) == 0); };
    std::vector<hs_profile_desc> new_raw(m->profiles, m->profiles + (m->profiles ? m->n_profiles : 0));
    for (auto &pr : new_raw) if (pr.kind == HS_PROF_STEP) pr.p[2] = 0.0;   /* a caller-side address, not part of the model */
    const bool same_model = E->have_model && E->ents.size() == n &&
        same_bytes(E->ents.data(), E->ents.size() * sizeof(hs_entity_desc), m->entities, (size_t)n * sizeof(hs_entity_desc)) &&
        same_bytes(E->backends.data(), E->backends.size() * 4, m->backends, (m->backends ? (size_t)m->n_backends : 0) * 4) &&
        same_bytes(E->key_table.data(), E->key_table.size() * 4, m->key_table, (m->key_table ? (size_t)m->key_population : 0) * 4) &&
        E->n_cells == m->n_cells &&
        same_bytes(E->cell_d0.data(), E->cell_d0.size() * 8, m->cell_d0, (size_t)m->n_cells * n * 8) &&
        same_bytes(E->cell_i0.data(), E->cell_i0.size() * 4, m->cell_i0, (size_t)m->n_cells * n * 4) &&
        same_bytes(E->profiles_raw.data(), E->profiles_raw.size() * sizeof(hs_profile_desc), new_raw.data(), new_raw.size() * sizeof(hs_profile_desc)) &&
        same_bytes(E->profile_table.data(), E->profile_table.size() * 8, m->profile_table, (m->profile_table ? (size_t)m->n_profile_table : 0) * 8) &&
        same_bytes(E->sketch_tab.data(), E->sketch_tab.size() * 4, m->sketch_tables, (m->sketch_tables ? (size_t)m->n_sketch_table : 0) * 4) &&
        same_bytes(E->key_cdf.data(), E->key_cdf.size() * 8, m->key_cdf, (m->key_cdf ? (size_t)m->n_key_cdf : 0) * 8);
    const bool keep_run = same_model && E->have_run && E->outbox_cap == m->outbox_cap && E->inbox_cap == m->inbox_cap;
    E->outbox_cap = m->outbox_cap; E->inbox_cap = m->inbox_cap;
    E->ents.assign(m->entities, m->entities + n);
    E->backends.assign(m->backends, m->backends + (m->backends ? m->n_backends : 0));
    E->key_table.assign(m->key_table, m->key_table + (m->key_table ? m->key_population : 0));
    E->n_cells = m->n_cells;
    E->profiles_raw = new_raw;
    E->profiles = new_raw;
    E->profile_table.assign(m->profile_table, m->profile_table + (m->profile_table ? m->n_profile_table : 0));
    E->cell_d0.clear(); E->cell_i0.clear();
    if (m->n_cells) {
        E->cell_d0.assign(m->cell_d0, m->cell_d0 + (size_t)m->n_cells * n);
        E->cell_i0.assign(m->cell_i0, m->cell_i0 + (size_t)m->n_cells * n);
    }
    auto up = [&](dev_buf &b, const void *src, size_t bytes) -> int {
        int r = b.ensure(bytes ? bytes : 16);
        if (r) return r;
        if (bytes) {
            cudaError_t e = cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, E->stream);
            if (e != cudaSuccess) return fail(HS_ERR_CUDA, "model upload failed: %s", cudaGetErrorString(e));
        }
        return 0;
    };
    E->sketch_tab.assign(m->sketch_tables, m->sketch_tables + (m->sketch_tables ? m->n_sketch_table : 0));
    E->sk_off.assign(n, 0); E->sk_moff.assign(n, 0);
    hs_sketch_layout_impl(m, E->sk_off.data(), E->sk_moff.data(), &E->sk_total, &E->sk_mtotal);
    /* device copy of the entity rows: the reserved d1 carries the server's index among the servers
     * (= its queue ring) or the SKETCH row's state offset, so the kernels get it with the row */
    std::vector<hs_entity_desc> dev_ents(E->ents);
    {
        int64_t k = 0;
        for (uint32_t i = 0; i < n; ++i) {
            hs_entity_desc &e = dev_ents[i];
            /* SERVER: its index among the queue rings; SKETCH: the offset of its state; CACHE_SERVER: both,
             * ring index in the low 24 bits, state offset above */
            const int64_t v = (e.kind == HS_ENT_SERVER) ? k++ : (e.kind == HS_ENT_SKETCH) ? (int64_t)E->sk_off[i]
                            : (e.kind == HS_ENT_CACHE_SERVER) ? ((k++) | ((int64_t)E->sk_off[i] << 24)) : -1;
            memcpy(&e.d1, &v, 8);
        }
    }
    if ((rc = up(E->d_sketch_tab, E->sketch_tab.data(), E->sketch_tab.size() * 4))) return rc;
    E->key_cdf.assign(m->key_cdf, m->key_cdf + (m->key_cdf ? m->n_key_cdf : 0));
    if ((rc = up(E->d_key_cdf, E->key_cdf.data(), E->key_cdf.size() * 8))) return rc;
    if ((rc = up(E->d_ents, dev_ents.data(), n * sizeof(hs_entity_desc)))) return rc;
    if ((rc = up(E->d_backends, E->backends.data(), E->backends.size() * 4))) return rc;
    if ((rc = up(E->d_key_table, E->key_table.data(), E->key_table.size() * 4))) return rc;
    if ((rc = up(E->d_cell_d0, E->cell_d0.data(), E->cell_d0.size() * 8))) return rc;
    if ((rc = up(E->d_cell_i0, E->cell_i0.data(), E->cell_i0.size() * 4))) return rc;
    if ((rc = up(E->d_profile_table, E->profile_table.data(), E->profile_table.size() * 8))) return rc;
    for (auto &pr : E->profiles)                       /* STEP rows carry the device address of their table */
        if (pr.kind == HS_PROF_STEP) {
            const uint64_t a = (uint64_t)(uintptr_t)((const double *)E->d_profile_table.p + (size_t)pr.p[0]);
            memcpy(&pr.p[2], &a, 8);
        }
    if ((rc = up(E->d_profiles, E->profiles.data(), E->profiles.size() * sizeof(hs_profile_desc)))) return rc;
    CUDA_TRY(cudaStreamSynchronize(E->stream));   /* host vectors may be reused by the caller's next upload */
    E->lane_ok = classify_lane(E);
    E->have_model = true;
    E->have_run = keep_run;
    return HS_OK;
}


int hs_run(hs_engine *E, const hs_run_params *p)
{
    if (!E || !p) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->have_model) return fail(HS_ERR_STATE, "hs_run before hs_model_upload");
    if (p->n_replicas == 0) return fail(HS_ERR_INVALID, "n_replicas must be > 0");
    if (p->end_ns < 0) return fail(HS_ERR_INVALID, "end_ns must be >= 0 (an explicit end_time is required)");
    if (p->replicas_per_cell == 0) return fail(HS_ERR_INVALID, "replicas_per_cell must be >= 1");
    CUDA_TRY(cudaSetDevice(E->device));

    if ((E->n_trace_arr || E->n_trace_svc) && p->n_replicas > E->trace_replicas)
        return fail(HS_ERR_INVALID, "hs_set_trace supplied draws for %u replicas, run asks for %u", E->trace_replicas, p->n_replicas);
    const bool linked = E->outbox_cap || E->inbox_cap || (p->flags & HS_RUN_LINKED);
    int engine = (int)p->engine;
    if (engine == 0) engine = E->lane_ok && !linked ? 2 : 3;
    if (engine < 1 || engine > 3) return fail(HS_ERR_INVALID, "unknown engine %d", engine);
    if (linked && engine != 3) return fail(HS_ERR_INVALID, "linked partitions run on the thread engine (engine 3)");
    if (engine == 2 && !E->lane_ok) return fail(HS_ERR_INVALID, "lane engine needs Source -> Server(concurrency <= 64) -> Sink|Counter");

    const uint32_t ring = p->queue_ring ? pow2_at_least(p->queue_ring) : engine == 2 ? 256 : 128;
    const bool want_hist = (p->flags & HS_RUN_HISTOGRAM) != 0;
    if (p->resume) {
        if (!E->have_run) return fail(HS_ERR_STATE, "resume without a previous run");
        const hs_run_params &q = E->last;
        if (q.n_replicas != p->n_replicas || q.seed != p->seed || q.seed_stride != p->seed_stride ||
            q.rid_base != p->rid_base || q.rid_stride != p->rid_stride || q.record_cap != p->record_cap ||
            q.sample_cap != p->sample_cap || q.service_cap != p->service_cap ||
            q.replica_index_base != p->replica_index_base || q.replicas_per_cell != p->replicas_per_cell ||
            engine != E->last_engine)
            return fail(HS_ERR_STATE, "resume must repeat the replica set, seeds and capacities of the paused run");
        if (want_hist != E->hist_on) return fail(HS_ERR_STATE, "resume must keep HS_RUN_HISTOGRAM");
        if (ring != E->last_ring) return fail(HS_ERR_STATE, "resume must keep queue_ring");
    }

    const uint32_t n = p->n_replicas;
    const uint32_t ne = (uint32_t)E->ents.size();
    int rc;
    if ((rc = E->d_summ.ensure((size_t)n * sizeof(hs_replica_summary)))) return rc;
    if ((rc = E->d_stats.ensure((size_t)n * ne * sizeof(hs_entity_stats)))) return rc;
    if ((rc = E->d_rec.ensure((size_t)n * p->record_cap * sizeof(hs_event_record)))) return rc;
    if ((rc = E->d_smp.ensure((size_t)n * p->sample_cap * sizeof(hs_sink_sample)))) return rc;
    if ((rc = E->d_svc.ensure((size_t)n * p->service_cap * sizeof(double)))) return rc;
    if (!p->resume) {
        CUDA_TRY(cudaMemsetAsync(E->d_stats.p, 0, (size_t)n * ne * sizeof(hs_entity_stats), E->stream));
        if (p->record_cap) CUDA_TRY(cudaMemsetAsync(E->d_rec.p, 0, (size_t)n * p->record_cap * sizeof(hs_event_record), E->stream));
        if (p->sample_cap) CUDA_TRY(cudaMemsetAsync(E->d_smp.p, 0, (size_t)n * p->sample_cap * sizeof(hs_sink_sample), E->stream));
        if (p->service_cap) CUDA_TRY(cudaMemsetAsync(E->d_svc.p, 0, (size_t)n * p->service_cap * sizeof(double), E->stream));
    }

    if (E->sk_total) {
        if ((rc = E->d_sketch.ensure((size_t)n * E->sk_total))) return rc;
        if (!p->resume) CUDA_TRY(cudaMemsetAsync(E->d_sketch.p, 0, (size_t)n * E->sk_total, E->stream));
    }
    if (want_hist) {
        if ((rc = E->d_hist.ensure((size_t)n * HS_HISTOGRAM_BINS * sizeof(uint32_t)))) return rc;
        if (!p->resume) CUDA_TRY(cudaMemsetAsync(E->d_hist.p, 0, (size_t)n * HS_HISTOGRAM_BINS * sizeof(uint32_t), E->stream));
    }
    E->hist_on = want_hist;
    if (E->outbox_cap || E->inbox_cap) {             /* linked partitions: per-replica outboxes / inboxes */
        if ((rc = E->d_outbox.ensure((size_t)n * std::max(1u, E->outbox_cap) * sizeof(hs_xevent)))) return rc;
        if ((rc = E->d_inbox.ensure((size_t)n * std::max(1u, E->inbox_cap) * sizeof(hs_xevent)))) return rc;
        if ((rc = E->d_outbox_n.ensure((size_t)n * 4 + 16))) return rc;
        if ((rc = E->d_inbox_n.ensure((size_t)n * 4 + 16))) return rc;
        if (!p->resume) {
            CUDA_TRY(cudaMemsetAsync(E->d_outbox_n.p, 0, (size_t)n * 4, E->stream));
            CUDA_TRY(cudaMemsetAsync(E->d_inbox_n.p, 0, (size_t)n * 4, E->stream));
        }
        E->link_replicas = n;
    }

    hs_kernel_run R;
    R.seed = p->seed; R.seed_stride = p->seed_stride; R.rid_base = p->rid_base; R.rid_stride = p->rid_stride;
    R.end_ns = p->end_ns; R.window_end_ns = p->window_end_ns;
    R.n_replicas = n; R.index_base = p->replica_index_base; R.replicas_per_cell = p->replicas_per_cell;
    R.record_cap = p->record_cap; R.sample_cap = p->sample_cap; R.service_cap = p->service_cap;
    R.ring = ring; R.resume = p->resume;
    R.max_events = p->max_events > 0 ? p->max_events : INT64_MAX;
    R.trace_arr = E->n_trace_arr ? (const double *)E->d_trace_arr.p : nullptr; R.n_trace_arr = E->n_trace_arr;
    R.trace_svc = E->n_trace_svc ? (const double *)E->d_trace_svc.p : nullptr; R.n_trace_svc = E->n_trace_svc;
    R.linked = (p->flags & HS_RUN_LINKED) ? 1u : 0u; R.lane_stride = 1; R.heap_top = 0;
    hs_kernel_out O;
    O.summaries = (hs_replica_summary *)E->d_summ.p; O.stats = (hs_entity_stats *)E->d_stats.p;
    O.records = p->record_cap ? (hs_event_record *)E->d_rec.p : nullptr;
    O.samples = p->sample_cap ? (hs_sink_sample *)E->d_smp.p : nullptr;
    O.service = p->service_cap ? (double *)E->d_svc.p : nullptr;
    O.hist = want_hist ? (uint32_t *)E->d_hist.p : nullptr;
    O.sketch = (uint8_t *)E->d_sketch.p;
    O.outbox = (hs_xevent *)E->d_outbox.p; O.outbox_n = (uint32_t *)E->d_outbox_n.p;
    O.inbox = (hs_xevent *)E->d_inbox.p; O.inbox_n = (uint32_t *)E->d_inbox_n.p;
    const bool want_hash = (p->flags & HS_RUN_ORDER_HASH) != 0;
    const bool want_rec = (p->record_cap | p->sample_cap | p->service_cap) != 0;
    rc = engine == 2 ? launch_lane(E, R, O, want_hash, want_rec)
       : engine == 3 ? launch_thread(E, R, O, want_hash, want_rec, linked)
       : launch_warp(E, R, O, want_hash, want_rec);
    if (rc) return rc;
    E->last = *p;
    E->last_engine = engine;
    E->last_ring = ring;
    E->have_run = true;
    return HS_OK;
}

int hs_set_trace(hs_engine *E, const double *arr, uint64_t n_arr, const double *svc, uint64_t n_svc, uint32_t n_replicas)
{
    if (!E) return fail(HS_ERR_INVALID, "engine is NULL");
    CUDA_TRY(cudaSetDevice(E->device));
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    E->n_trace_arr = E->n_trace_svc = 0; E->trace_replicas = 0;
    if ((!arr || !n_arr) && (!svc || !n_svc)) return HS_OK;
    if (n_replicas == 0) return fail(HS_ERR_INVALID, "n_replicas must be > 0");
    int rc;
    if (arr && n_arr) {
        if ((rc = E->d_trace_arr.ensure((size_t)n_replicas * n_arr * 8))) return rc;
        CUDA_TRY(cudaMemcpy(E->d_trace_arr.p, arr, (size_t)n_replicas * n_arr * 8, cudaMemcpyHostToDevice));
        E->n_trace_arr = n_arr;
    }
    if (svc && n_svc) {
        if ((rc = E->d_trace_svc.ensure((size_t)n_replicas * n_svc * 8))) return rc;
        CUDA_TRY(cudaMemcpy(E->d_trace_svc.p, svc, (size_t)n_replicas * n_svc * 8, cudaMemcpyHostToDevice));
        E->n_trace_svc = n_svc;
    }
    E->trace_replicas = n_replicas;
    return HS_OK;
}

int hs_sync(hs_engine *E)
{
    if (!E) return fail(HS_ERR_INVALID, "engine is NULL");
    CUDA_TRY(cudaSetDevice(E->device));
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    return HS_OK;
}

int hs_last_run_ms(hs_engine *E, float *ms)
{
    if (!E || !ms) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->have_run) return fail(HS_ERR_STATE, "no run yet");
    CUDA_TRY(cudaEventSynchronize(E->ev1));
    CUDA_TRY(cudaEventElapsedTime(ms, E->ev0, E->ev1));
    return HS_OK;
}

int hs_launch_count(hs_engine *E, uint64_t *n)
{
    if (!E || !n) return fail(HS_ERR_INVALID, "NULL argument");
    *n = E->launches;
    return HS_OK;
}

int hs_last_launch(hs_engine *E, hs_launch_info *out)
{
    if (!E || !out) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->last_launch.engine) return fail(HS_ERR_STATE, "no run yet");
    *out = E->last_launch;
    return HS_OK;
}

int hs_read_outputs(hs_engine *E, const hs_outputs *out)
{
    if (!E || !out) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->have_run) return fail(HS_ERR_STATE, "no run yet");
    CUDA_TRY(cudaSetDevice(E->device));
    const hs_run_params &p = E->last;
    const size_t n = p.n_replicas, ne = E->ents.size();
    if (out->summaries) CUDA_TRY(cudaMemcpyAsync(out->summaries, E->d_summ.p, n * sizeof(hs_replica_summary), cudaMemcpyDeviceToHost, E->stream));
    if (out->entity_stats) CUDA_TRY(cudaMemcpyAsync(out->entity_stats, E->d_stats.p, n * ne * sizeof(hs_entity_stats), cudaMemcpyDeviceToHost, E->stream));
    if (out->records && p.record_cap) CUDA_TRY(cudaMemcpyAsync(out->records, E->d_rec.p, n * p.record_cap * sizeof(hs_event_record), cudaMemcpyDeviceToHost, E->stream));
    if (out->sink_samples && p.sample_cap) CUDA_TRY(cudaMemcpyAsync(out->sink_samples, E->d_smp.p, n * p.sample_cap * sizeof(hs_sink_sample), cudaMemcpyDeviceToHost, E->stream));
    if (out->histograms && E->hist_on) CUDA_TRY(cudaMemcpyAsync(out->histograms, E->d_hist.p, n * HS_HISTOGRAM_BINS * sizeof(uint32_t), cudaMemcpyDeviceToHost, E->stream));
    if (out->service_samples && p.service_cap) CUDA_TRY(cudaMemcpyAsync(out->service_samples, E->d_svc.p, n * p.service_cap * sizeof(double), cudaMemcpyDeviceToHost, E->stream));
    if (out->sketches && E->sk_total) CUDA_TRY(cudaMemcpyAsync(out->sketches, E->d_sketch.p, n * E->sk_total, cudaMemcpyDeviceToHost, E->stream));
    /* linked partitions: what the last barrier delivered is scheduled on the receiver (Simulation.schedule = heap push,
     * coordinator.py:222) whether or not another window follows -- those events wait in the inbox here and are part of
     * the pending-event count like everything else in the reference's heap */
    std::vector<uint32_t> inbox_n;
    if (out->summaries && E->inbox_cap && E->link_replicas == n) {
        inbox_n.resize(n);
        CUDA_TRY(cudaMemcpyAsync(inbox_n.data(), E->d_inbox_n.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, E->stream));
    }
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    for (size_t r = 0; r < inbox_n.size(); ++r) out->summaries[r].heap_left += (int32_t)inbox_n[r];
    return HS_OK;
}

int hs_sketch_layout(const hs_model_desc *m, uint64_t *per_replica, uint64_t *merged, uint64_t *total, uint64_t *merged_total)
{
    if (!m || !m->entities) return fail(HS_ERR_INVALID, "model is NULL");
    hs_sketch_layout_impl(m, per_replica, merged, total, merged_total);
    return HS_OK;
}

int hs_read_sketches(hs_engine *E, void *merged, uint64_t merged_bytes)
{
    if (!E || !merged) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->have_run) return fail(HS_ERR_STATE, "no run yet");
    if (merged_bytes != E->sk_mtotal) return fail(HS_ERR_INVALID, "merged image is %llu bytes, caller passed %llu", (unsigned long long)E->sk_mtotal, (unsigned long long)merged_bytes);
    if (!E->sk_mtotal) return HS_OK;
    CUDA_TRY(cudaSetDevice(E->device));
    int rc;
    if ((rc = E->d_sketch_merged.ensure(E->sk_mtotal))) return rc;
    const uint32_t n = E->last.n_replicas;
    CUDA_TRY(cudaMemsetAsync(E->d_sketch_merged.p, 0, E->sk_mtotal, E->stream));
    for (size_t i = 0; i < E->ents.size(); ++i) {
        const hs_entity_desc &e = E->ents[i];
        if (e.kind != HS_ENT_SKETCH) continue;
        const uint8_t *src = (const uint8_t *)E->d_sketch.p + E->sk_off[i];
        uint8_t *dst = (uint8_t *)E->d_sketch_merged.p + E->sk_moff[i];
        if (e.i0 == HS_SK_HLL) {
            const uint32_t words = (1u << e.i2) / 4u;
            hs_sketch_merge_hll_kernel<<<(words + 127) / 128, 128, 0, E->stream>>>(src, E->sk_total, n, words, (uint32_t *)dst);
        } else if (e.i0 == HS_SK_BLOOM) {
            const uint32_t words = (uint32_t)(hs_sketch_row_bytes(&e) / 4u);
            hs_sketch_merge_or_kernel<<<(words + 127) / 128, 128, 0, E->stream>>>(src, E->sk_total, n, words, (uint32_t *)dst);
        } else if (e.i0 == HS_SK_TOPK || e.i0 == HS_SK_TDIGEST || e.i0 == HS_SK_RESERVOIR) {
            continue;                                   /* no merged image: these merges are sequential, done by the host layer */
        } else {
            const uint32_t cells = (uint32_t)e.i2 * (uint32_t)e.i3;
            hs_sketch_merge_cms_kernel<<<(cells + 127) / 128, 128, 0, E->stream>>>(src, E->sk_total, n, cells, (unsigned long long *)dst);
        }
        CUDA_TRY(cudaGetLastError());
        E->launches += 1;
    }
    CUDA_TRY(cudaMemcpyAsync(merged, E->d_sketch_merged.p, E->sk_mtotal, cudaMemcpyDeviceToHost, E->stream));
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    return HS_OK;
}

static int compute_totals(hs_engine *E)
{
    const hs_run_params &p = E->last;
    int rc;
    const int blocks = 256;
    if ((rc = E->d_partials.ensure((size_t)blocks * sizeof(hs_totals)))) return rc;
    if ((rc = E->d_totals.ensure(sizeof(hs_totals)))) return rc;
    hs_totals_partial_kernel<<<blocks, 256, 0, E->stream>>>(
        (const hs_replica_summary *)E->d_summ.p, (const hs_entity_stats *)E->d_stats.p,
        (const hs_entity_desc *)E->d_ents.p, p.n_replicas, (uint32_t)E->ents.size(), (hs_totals *)E->d_partials.p);
    CUDA_TRY(cudaGetLastError());
    hs_totals_final_kernel<<<1, 32, 0, E->stream>>>((const hs_totals *)E->d_partials.p, blocks, (hs_totals *)E->d_totals.p);
    CUDA_TRY(cudaGetLastError());
    E->launches += 2;
    return HS_OK;
}

int hs_read_totals(hs_engine *E, hs_totals *out)
{
    if (!E || !out) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->have_run) return fail(HS_ERR_STATE, "no run yet");
    CUDA_TRY(cudaSetDevice(E->device));
    int rc = compute_totals(E);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, E->d_totals.p, sizeof(hs_totals), cudaMemcpyDeviceToHost, E->stream));
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    return HS_OK;
}

int hs_read_cell_totals(hs_engine *E, hs_cell_totals *out, uint32_t n_cells)
{
    if (!E || !out || n_cells == 0) return fail(HS_ERR_INVALID, "bad argument");
    if (!E->have_run) return fail(HS_ERR_STATE, "no run yet");
    CUDA_TRY(cudaSetDevice(E->device));
    const hs_run_params &p = E->last;
    int rc;
    if ((rc = E->d_cell_totals.ensure((size_t)n_cells * sizeof(hs_cell_totals)))) return rc;
    hs_cell_totals_kernel<<<n_cells, 128, 0, E->stream>>>(
        (const hs_replica_summary *)E->d_summ.p, (const hs_entity_stats *)E->d_stats.p, (const hs_entity_desc *)E->d_ents.p,
        E->hist_on ? (const uint32_t *)E->d_hist.p : nullptr, p.n_replicas, (uint32_t)E->ents.size(),
        p.replica_index_base, p.replicas_per_cell, n_cells, (hs_cell_totals *)E->d_cell_totals.p);
    CUDA_TRY(cudaGetLastError());
    E->launches += 1;
    CUDA_TRY(cudaMemcpyAsync(out, E->d_cell_totals.p, (size_t)n_cells * sizeof(hs_cell_totals), cudaMemcpyDeviceToHost, E->stream));
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    return HS_OK;
}

int hs_totals_device_ptr(hs_engine *E, void **ptr)
{
    if (!E || !ptr) return fail(HS_ERR_INVALID, "NULL argument");
    if (!E->have_run) return fail(HS_ERR_STATE, "no run yet");
    CUDA_TRY(cudaSetDevice(E->device));
    int rc = compute_totals(E);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    *ptr = E->d_totals.p;
    return HS_OK;
}

/* ---- linked partitions: the window barrier (parallel/coordinator.py:182-227) ---------------------------- */
#define HS_MAX_LINKS_ 16
struct hs_link_dev { int32_t kind, stream; double mean_s, loss; hs_xevent *inbox; uint32_t *inbox_n; uint32_t inbox_cap, pad; };
struct hs_links_dev { hs_link_dev l[HS_MAX_LINKS_]; };

struct hs_coordinator {
    int device = 0; cudaStream_t stream = nullptr;
    uint32_t n = 0, n_streams = 1;
    uint64_t seed = 0, seed_stride = 0; uint32_t rid_base = 0, rid_stride = 0, index_base = 0;
    dev_buf d_loss_draws, d_lat_draws, d_counts;      /* uint64[n], uint64[n][n_streams], uint64[3][n] */
};

/* one thread per replica: its outbox in emission order -- one loss draw when the link loses packets, then
 * event.time = send_time + latency.sample(), then Simulation.schedule(event) = a slot of the destination's inbox */
__global__ void hs_exchange_kernel(const hs_xevent *__restrict__ outbox, uint32_t *__restrict__ outbox_n, uint32_t ocap,
                                   const hs_entity_desc *__restrict__ src_ents, hs_links_dev LK, uint32_t n, uint32_t n_streams,
                                   uint64_t seed0, uint64_t seed_stride, uint32_t rid_base, uint32_t rid_stride, uint32_t index_base,
                                   uint64_t *__restrict__ loss_draws, uint64_t *__restrict__ lat_draws, uint64_t *__restrict__ counts)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint32_t g = index_base + r;
    const uint64_t seed = seed0 + (uint64_t)g * seed_stride;
    const uint32_t rid = rid_base + g * rid_stride;
    const uint32_t cnt = outbox_n[r];
    uint64_t nl = loss_draws[r], delivered = 0, lost = 0, over = 0;
    for (uint32_t k = 0; k < cnt; ++k) {
        const hs_xevent x = outbox[(size_t)r * ocap + k];
        const hs_entity_desc row = src_ents[x.ent];
        const hs_link_dev &L = LK.l[row.i0];
        if (L.loss > 0.0 && hs_uniform(seed, rid, HS_STREAM_LINK_LOSS, nl++) < L.loss) { lost++; continue; }
        int64_t lat;
        if (L.kind == HS_SVC_EXPONENTIAL) {
            const uint64_t d = lat_draws[(size_t)r * n_streams + L.stream]++;
            lat = hs_exp_latency_ns(hs_uniform(seed, rid, HS_STREAM_LINK_LATENCY | ((uint32_t)L.stream << 8), d), HS_DIV(1.0, L.mean_s));
        } else lat = hs_seconds_to_ns(L.mean_s);
        const uint32_t m = L.inbox_n[r];
        if (m >= L.inbox_cap) { over++; continue; }
        hs_xevent y = x; y.time_ns = x.time_ns + lat; y.ent = row.i1;
        L.inbox[(size_t)r * L.inbox_cap + m] = y;
        L.inbox_n[r] = m + 1u;
        delivered++;
    }
    outbox_n[r] = 0u;
    loss_draws[r] = nl;
    counts[r] += delivered; counts[(size_t)n + r] += lost; counts[2 * (size_t)n + r] += over;
}

int hs_coordinator_create(int device, void *cuda_stream, uint32_t n_replicas, uint32_t n_streams,
                          uint64_t seed, uint64_t seed_stride, uint32_t rid_base, uint32_t rid_stride,
                          uint32_t replica_index_base, hs_coordinator **out)
{
    if (!out || !n_replicas) return fail(HS_ERR_INVALID, "hs_coordinator_create: bad arguments");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return fail(HS_ERR_NO_DEVICE, "no CUDA device available");
    if (device < 0 || device >= count) return fail(HS_ERR_INVALID, "device %d out of range", device);
    CUDA_TRY(cudaSetDevice(device));
    hs_coordinator *c = new hs_coordinator();
    c->device = device; c->stream = (cudaStream_t)cuda_stream; c->n = n_replicas; c->n_streams = n_streams ? n_streams : 1u;
    c->seed = seed; c->seed_stride = seed_stride; c->rid_base = rid_base; c->rid_stride = rid_stride; c->index_base = replica_index_base;
    int rc;
    if ((rc = c->d_loss_draws.ensure((size_t)n_replicas * 8)) || (rc = c->d_lat_draws.ensure((size_t)n_replicas * c->n_streams * 8)) ||
        (rc = c->d_counts.ensure((size_t)n_replicas * 24))) { delete c; return rc; }
    CUDA_TRY(cudaMemsetAsync(c->d_loss_draws.p, 0, (size_t)n_replicas * 8, c->stream));
    CUDA_TRY(cudaMemsetAsync(c->d_lat_draws.p, 0, (size_t)n_replicas * c->n_streams * 8, c->stream));
    CUDA_TRY(cudaMemsetAsync(c->d_counts.p, 0, (size_t)n_replicas * 24, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    *out = c;
    return HS_OK;
}

void hs_coordinator_destroy(hs_coordinator *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    c->d_loss_draws.release(); c->d_lat_draws.release(); c->d_counts.release();
    delete c;
}

int hs_coordinator_exchange(hs_coordinator *c, hs_engine *src, uint32_t n_links, const hs_link_desc *links, hs_engine *const *dsts)
{
    if (!c || !src) return fail(HS_ERR_INVALID, "hs_coordinator_exchange: NULL handle");
    if (n_links > HS_MAX_LINKS_ || (n_links && (!links || !dsts))) return fail(HS_ERR_INVALID, "hs_coordinator_exchange: at most %d links", HS_MAX_LINKS_);
    if (!src->have_run || !src->outbox_cap) return HS_OK;              /* nothing can have been sent */
    if (src->link_replicas != c->n) return fail(HS_ERR_STATE, "the coordinator was created for %u replicas, the partition ran %u", c->n, src->link_replicas);
    CUDA_TRY(cudaSetDevice(c->device));
    hs_links_dev LK; memset(&LK, 0, sizeof LK);
    bool foreign = src->stream != c->stream;          /* everything on one stream: the window loop needs no host synchronisation */
    for (const hs_entity_desc &e : src->ents)
        if (e.kind == HS_ENT_REMOTE && (uint32_t)e.i0 >= n_links) return fail(HS_ERR_INVALID, "a REMOTE row uses link slot %d of %u", e.i0, n_links);
    for (uint32_t k = 0; k < n_links; ++k) {
        hs_engine *D = dsts[k];
        if (!D || D == src) return fail(HS_ERR_INVALID, "link %u: bad destination engine", k);
        if (D->device != src->device) return fail(HS_ERR_INVALID, "link %u: the partitions of one replica set live on one device", k);
        if (!D->inbox_cap || !D->have_run || D->link_replicas != c->n) return fail(HS_ERR_STATE, "link %u: the destination has no inbox or has not run these replicas", k);
        if (links[k].latency_kind != HS_SVC_CONSTANT && links[k].latency_kind != HS_SVC_EXPONENTIAL) return fail(HS_ERR_INVALID, "link %u: bad latency kind", k);
        if (!(links[k].latency_mean_s >= 0.0) || !(links[k].packet_loss >= 0.0 && links[k].packet_loss < 1.0)) return fail(HS_ERR_INVALID, "link %u: latency must be >= 0 and packet_loss in [0, 1) (parallel/link.py:45-52)", k);
        if (links[k].stream < 0 || (uint32_t)links[k].stream >= c->n_streams) return fail(HS_ERR_INVALID, "link %u: latency stream %d of %u", k, links[k].stream, c->n_streams);
        for (const hs_entity_desc &e : src->ents)
            if (e.kind == HS_ENT_REMOTE && (uint32_t)e.i0 == k) {
                if ((size_t)e.i1 >= D->ents.size()) return fail(HS_ERR_INVALID, "link %u: destination entity %d out of range", k, e.i1);
                const int dk = D->ents[e.i1].kind;
                if (dk == HS_ENT_SOURCE || dk == HS_ENT_PROBE || dk == HS_ENT_REMOTE) return fail(HS_ERR_INVALID, "link %u: destination entity %d cannot receive requests", k, e.i1);
            }
        LK.l[k].kind = links[k].latency_kind; LK.l[k].stream = links[k].stream; LK.l[k].mean_s = links[k].latency_mean_s;
        LK.l[k].loss = links[k].packet_loss; LK.l[k].inbox = (hs_xevent *)D->d_inbox.p; LK.l[k].inbox_n = (uint32_t *)D->d_inbox_n.p;
        LK.l[k].inbox_cap = D->inbox_cap;
        if (D->stream != c->stream) { foreign = true; CUDA_TRY(cudaStreamSynchronize(D->stream)); }
    }
    if (src->stream != c->stream) CUDA_TRY(cudaStreamSynchronize(src->stream));
    const uint32_t threads = 128, blocks = (c->n + threads - 1) / threads;
    hs_exchange_kernel<<<blocks, threads, 0, c->stream>>>((const hs_xevent *)src->d_outbox.p, (uint32_t *)src->d_outbox_n.p, src->outbox_cap,
        (const hs_entity_desc *)src->d_ents.p, LK, c->n, c->n_streams, c->seed, c->seed_stride, c->rid_base, c->rid_stride, c->index_base,
        (uint64_t *)c->d_loss_draws.p, (uint64_t *)c->d_lat_draws.p, (uint64_t *)c->d_counts.p);
    CUDA_TRY(cudaGetLastError());
    if (foreign) CUDA_TRY(cudaStreamSynchronize(c->stream));      /* a partition on another stream must not run ahead of the barrier */
    src->launches += 1;
    return HS_OK;
}

int hs_coordinator_read(hs_coordinator *c, uint64_t *delivered, uint64_t *lost, uint64_t *overflowed)
{
    if (!c) return fail(HS_ERR_INVALID, "hs_coordinator_read: NULL handle");
    CUDA_TRY(cudaSetDevice(c->device));
    const size_t nb = (size_t)c->n * 8;
    if (delivered) CUDA_TRY(cudaMemcpyAsync(delivered, c->d_counts.p, nb, cudaMemcpyDeviceToHost, c->stream));
    if (lost) CUDA_TRY(cudaMemcpyAsync(lost, (const uint8_t *)c->d_counts.p + nb, nb, cudaMemcpyDeviceToHost, c->stream));
    if (overflowed) CUDA_TRY(cudaMemcpyAsync(overflowed, (const uint8_t *)c->d_counts.p + 2 * nb, nb, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return HS_OK;
}

static int read_box(hs_engine *E, const dev_buf &box, const dev_buf &cnt, uint32_t cap, hs_xevent *buf, uint32_t *counts)
{
    if (!E || !E->have_run) return fail(HS_ERR_STATE, "no run to read");
    CUDA_TRY(cudaSetDevice(E->device));
    if (!cap) return HS_OK;
    if (buf) CUDA_TRY(cudaMemcpyAsync(buf, box.p, (size_t)E->link_replicas * cap * sizeof(hs_xevent), cudaMemcpyDeviceToHost, E->stream));
    if (counts) CUDA_TRY(cudaMemcpyAsync(counts, cnt.p, (size_t)E->link_replicas * 4, cudaMemcpyDeviceToHost, E->stream));
    CUDA_TRY(cudaStreamSynchronize(E->stream));
    return HS_OK;
}
int hs_read_outbox(hs_engine *E, hs_xevent *buf, uint32_t *counts) { return read_box(E, E->d_outbox, E->d_outbox_n, E ? E->outbox_cap : 0, buf, counts); }
int hs_read_inbox(hs_engine *E, hs_xevent *buf, uint32_t *counts) { return read_box(E, E->d_inbox, E->d_inbox_n, E ? E->inbox_cap : 0, buf, counts); }

} /* extern "C" */
