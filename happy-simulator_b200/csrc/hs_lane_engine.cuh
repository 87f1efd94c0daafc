/* hs_lane_engine.cuh -- "lane engine": one THREAD per replica for the
 * single-server topology  Source -> Server(concurrency c) -> Sink|Counter|nothing
 * (BASELINE.json configs[0], configs[1] -- the headline M/M/1 ensemble -- and the M/M/c
 * sweep of configs[4]).
 *
 * Why a lane and not a warp per replica: the whole future-event list of this
 * topology is {next SourceEvent, at most one ProcessContinuation, a handful of
 * same-timestamp protocol events}, i.e. a few registers.  Giving each replica a
 * lane keeps all 32 lanes of a warp doing useful event work; a warp per replica
 * would leave 31 lanes idle in every handler.  (The general "warp engine",
 * hs_warp_engine.cuh, covers models whose state does not fit a lane.)
 *
 * Exactness.  The loop below is the reference's pop-invoke-push loop
 * (happysimulator/core/simulation.py:449-505) with the future-event list held as
 *   T   the pending SourceEvent                     (time tT, sort index iT)
 *   C   the pending ProcessContinuations (<= c): the earliest in registers
 *       (time tC, sort index iC), the others in a small per-lane binary heap in HBM
 *   nowq  events created at the current timestamp   (sort index, kind, payload)
 * Two execution paths produce the SAME processed-event sequence:
 *   - generic_step(): pops the (time, sort_index)-minimum of T, C and nowq and
 *     runs that one handler, exactly like the oracle;
 *   - the fused arrival / completion chains: when nowq is empty and neither T
 *     nor C shares the timestamp being processed, every event a handler creates
 *     at `now` is provably the next pop (ties between them are resolved by the
 *     creation order, which the straight-line code follows; the re-pushed payload
 *     keeps its OLD index and therefore sorts first, queue_driver.py:86-90), so the
 *     chain TICK -> ENQUEUE -> NOTIFY -> POLL -> DELIVER -> WORKER or
 *     CONTINUATION -> SINK -> POLL -> DELIVER -> WORKER is executed inline with the
 *     same counters, indices, hash and records.
 * Same-nanosecond ties (SURVEY.md Appendix A.12) fall back to generic_step().
 *
 * Random draws.  Every draw is a pure function of (seed, replica, stream, draw
 * index), so the expensive part of a draw -- Philox block, log, the IEEE
 * divisions of arrival_time_provider.py:77 and exponential.py:43-45 -- does not
 * depend on simulation state and is computed AHEAD of its use, in warp-converged
 * "refill rounds": whenever any lane of the warp has run out of arrival or
 * service draws, all 32 lanes generate their next Philox pair of each stream
 * (four independent log/divide chains per lane: full lane utilisation and
 * instruction-level parallelism) into per-lane ring buffers in shared memory
 * ([slot][lane] layout: conflict-free whatever slot each lane is at).  The
 * divergent event loop then only pops a precomputed value:
 *     arrival  A_k = Instant.from_seconds(A_{k-1} / 1e9 + target_k / rate), the k-th
 *              SourceEvent time itself: the arrival process of a Source does not
 *              depend on anything downstream (arrival_time_provider.py:66-82)
 *     service  (svc_s, delta_ns) = (to_seconds(dur), int(svc_s * 1e9))
 * which is bit-identical to drawing at the point of use because the reference
 * consumes each stream strictly in draw-index order.
 *
 * Queue.  Items wait in a per-replica ring in HBM; the item the next POLL will
 * deliver (FIFO head / LIFO tail) is also kept in registers and re-loaded right
 * after every pop, one whole service time before it is needed, so the ring load
 * latency is off the critical path.  Recorder streams (event records, Sink and
 * service samples) are written with streaming stores (st.global.cs) so they do
 * not evict the queue rings from L2.
 *
 * Reference handlers restated (paths under /root/reference/happysimulator):
 *   load/source.py:142-180, load/arrival_time_provider.py:66-82,
 *   components/queue.py:122-166, components/queue_driver.py:66-99,
 *   components/server/server.py:202-273, components/server/concurrency.py:100-128,
 *   components/common.py:36-44,92-95, core/event.py:277-325,465-533.
 */
#ifndef HS_LANE_ENGINE_CUH
#define HS_LANE_ENGINE_CUH

#include "hs_sampler.h"
#include "hs_profile.h"
#include "hs_kernel_params.cuh"
#include "hs_buckets.cuh"

#define HS_NOW_CAP 8
#define HS_LANE_THREADS 64
#define HS_DRAW_BUF_SUMMARY 16  /* precomputed draws per stream per lane (even)            */
#define HS_DRAW_BUF_RECORD 8    /* ... when the recorder staging shares the shared memory  */
#define HS_ARR_BUF_RECORD 7     /* arrival draws per lane of the recorder kernels: 7, not 8, keeps their shared
                                   memory at 28 160 B, at which 8 blocks of 64 threads fit an SM */
#define HS_STAGE 16             /* staged event records per lane (recorder kernels)        */
#define HS_FLUSH 8              /* records per flush: 8 x 16 B = one 128 B line            */
#define HS_SMP_GROUP 4          /* Sink samples per flush: 4 x 16 B = one 64 B chunk        */
#define HS_SVC_CHUNK 8          /* service times per chunk: 8 x 8 B = 64 B (= HS_DRAW_BUF_RECORD) */
#define HS_LF_HASH 1      /* maintain the order hash                         */
#define HS_LF_REC 2       /* write event records / sink / service samples    */
#define HS_LF_PROFILE 4   /* non-constant rate profile (Simpson + Brent path) */
#define HS_LF_SIMPLE 8    /* compile-time model: Poisson source without stop_after, exponential FIFO server with an
                             unbounded queue, Sink downstream, Philox draws -- the BASELINE configs[0]/[1] shape */
#define HS_LF_BUCKETS 16  /* time buckets of the Sink samples (hs_set_buckets; the Sink is bucketed row 0); compiled
                             without HS_LF_REC only */
#define HS_LF_BUCKET_PCT 32 /* with HS_LF_BUCKETS: the buckets' p50 / p99 (hs_set_bucket_percentiles) */

/* The flag words (F < 64) hs_lane_kernel is built for (hs_engine.cu launches it through a table indexed by the flag
 * word): a SIMPLE model has no profile, BUCKETS never comes with the recorder, BUCKET_PCT only with BUCKETS. */
constexpr bool hs_lane_built(int F)
{
    return !((F & HS_LF_SIMPLE) && (F & HS_LF_PROFILE)) && !((F & HS_LF_BUCKETS) && (F & HS_LF_REC)) &&
           (!(F & HS_LF_BUCKET_PCT) || (F & HS_LF_BUCKETS));
}

struct hs_now_ev {        /* an event created at the current timestamp       */
    uint64_t idx;         /* Event._sort_index                               */
    int64_t created;      /* context["created_at"]                           */
    uint64_t payload_idx; /* DELIVER: sort index of the payload it carries   */
    int32_t kind;         /* HS_EV_*                                         */
    int32_t pad;
};

struct hs_cont {          /* a pending ProcessContinuation (service in progress)  */
    int64_t t;            /* resume time                                      */
    uint64_t idx;         /* its _sort_index                                  */
    int64_t created;      /* context["created_at"] of the request served      */
    double svc_s;         /* the service time the generator yielded           */
};

struct hs_ring_entry {    /* one queued request (FIFOQueue/LIFOQueue item)   */
    int64_t created;      /* context["created_at"]                           */
    uint64_t idx;         /* the queued Event's _sort_index                  */
};

struct __align__(16) hs_lane_state {   /* persisted between windows (512 B)  */
    int64_t now; uint64_t ctr; int64_t processed; uint64_t hash;
    int64_t tT; uint64_t iT; uint64_t arr_draws; int64_t gen_count; int64_t prov_count;
    int64_t tC; uint64_t iC; double svc_s; int64_t c_created;
    uint64_t svc_draws; int64_t accepted, dropped, completed, rejected; double total_service;
    int64_t received; double sum, sumsq, mn, mx;
    uint32_t q_head, q_len; int32_t active; uint32_t status;
    int64_t n_smp, n_svc; int32_t now_n; int32_t has_c;
    int32_t done; uint32_t rec_pos; double comp; uint32_t smp_pos, svc_pos; int64_t skipped;
    hs_now_ev nowq[HS_NOW_CAP];
};

struct hs_lane_model {
    int32_t src_id, srv_id, dst_id;   /* entity ids (dst_id < 0: no downstream) */
    int32_t dst_kind;                 /* HS_ENT_SINK / HS_ENT_COUNTER / 0       */
    int32_t arr_kind, svc_kind, policy, n_entities;
    int64_t capacity, stop_after;
    double rate, mean;
    uint32_t n_cells, pad;
    const double *cell_d0;            /* device pointers or NULL                */
    hs_profile_desc prof;             /* the Source's rate profile                */
    const int32_t *cell_i0;           /* per-cell concurrency override or NULL    */
    int32_t concurrency, c_max;       /* FixedConcurrency limit; heap stride      */
    int32_t has_profile, pad2;        /* 0: ConstantRateProfile fast path         */
};

/* next arrival of a constant-rate profile, with the reference's "time travel" outcome
 * folded in: if the computed time is earlier than the current one the SourceEvent would be
 * popped and skipped and the Source never ticks again (INT64_MAX). */
template <bool PROFILE>
__device__ __forceinline__ int64_t hs_lane_next_arrival(int64_t t, double target, double rate, double rate_recip,
                                                        const hs_profile_desc *prof)
{
    if (t >= HS_T_EXHAUSTED) return t;              /* dead / exhausted source stays so */
    int64_t n;
    if (PROFILE) n = hs_next_arrival_profile_ns(prof, t, target);
    else n = hs_next_arrival_ns_r(t, target, rate, rate_recip);
    if (n == HS_T_EXHAUSTED) return n;              /* RuntimeError: no further SourceEvent object */
    return n < t ? INT64_MAX : n;
}

/* lane of the k-th lowest set bit of mask (k < K; 32: fewer than k + 1 bits set), the owner a lane serves in a round of
 * the recorder's warp-wide flushes.  The same result as min(__fns(mask, 0, k + 1), 32), in K - 1 predicated steps and
 * one find-first: __fns is a branchy binary search of about 50 dependent instructions, run once per round of every
 * flush, where it made up most of the flush's latency. */
template <uint32_t K>
__device__ __forceinline__ uint32_t hs_kth_set_lane(uint32_t mask, uint32_t k)
{
#pragma unroll
    for (uint32_t q = 0; q + 1 < K; ++q) mask = q < k ? mask & (mask - 1u) : mask;
    return mask ? (uint32_t)(__ffs((int)mask) - 1) : 32u;
}

template <int FLAGS>
__global__ void __launch_bounds__(HS_LANE_THREADS, 7)
hs_lane_kernel(hs_lane_model M, hs_kernel_run P, hs_lane_state *__restrict__ states,
               hs_ring_entry *__restrict__ rings, hs_cont *__restrict__ conts, hs_kernel_out O,
               typename hs_bucket_args_of<(FLAGS & HS_LF_BUCKETS) != 0, (FLAGS & HS_LF_BUCKET_PCT) != 0>::type BK)
{
    constexpr uint32_t HS_DRAW_BUF = (FLAGS & HS_LF_REC) ? HS_DRAW_BUF_RECORD : HS_DRAW_BUF_SUMMARY;
    constexpr uint32_t ARR_BUF = (FLAGS & HS_LF_REC) ? HS_ARR_BUF_RECORD : HS_DRAW_BUF;
    constexpr uint32_t STAGE_ROWS = (FLAGS & HS_LF_REC) ? HS_STAGE : 1;
    static_assert(!(FLAGS & HS_LF_REC) || HS_DRAW_BUF == HS_SVC_CHUNK, "a service chunk is the whole draw buffer");
    __shared__ int64_t sh_t[ARR_BUF][HS_LANE_THREADS];           /* arrival times A_k (ns)          */
    __shared__ double sh_svc[HS_DRAW_BUF][HS_LANE_THREADS];      /* service: Duration.to_seconds()  */
    /* recorder staging, [slot][lane]: a lane writes only its own 16-byte column, so the per-event writes do
     * not conflict, whatever slot each lane is at.  Full 128-byte groups (8 records) and full 64-byte groups
     * of Sink samples (4) are written by the whole warp at the top of the loop, several groups per store.
     * The first three samples of a group wait in sh_smp; the fourth, which makes the group full, waits in row
     * (st_fl - 1) % HS_STAGE of the record staging: at most 7 + 6 records are staged between two flushes,
     * so that row is free from the sample's store to the next flush.  Service times need no staging: a
     * whole 64-byte chunk of them is the draw buffer sh_svc itself (the refill round writes it). */
    static_assert(HS_STAGE >= (HS_FLUSH - 1) + 6 + 1, "a free record-staging row for the fourth sample of a group");
    __shared__ __align__(16) uint4 sh_rec[STAGE_ROWS][HS_LANE_THREADS];
    __shared__ __align__(16) uint4 sh_smp[(FLAGS & HS_LF_REC) ? HS_SMP_GROUP - 1 : 1][HS_LANE_THREADS];
    __shared__ __align__(16) hs_ring_entry sh_head[HS_LANE_THREADS];  /* next item to deliver      */
    const uint32_t tid = threadIdx.x;
    uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = r < P.n_replicas;
    if (!valid) r = P.n_replicas - 1;      /* idle lane of the last warp: votes only, stores nothing */

    const uint32_t gidx = P.index_base + r;
    const uint64_t seed = P.seed + (uint64_t)gidx * P.seed_stride;
    const uint32_t rid = P.rid_base + gidx * P.rid_stride;
    const uint32_t sid_arr = HS_STREAM_ARRIVAL | ((uint32_t)M.src_id << 8);
    const uint32_t sid_svc = HS_STREAM_SERVICE | ((uint32_t)M.srv_id << 8);

    double rate = M.rate, mean = M.mean;
    int32_t c_rt = M.concurrency;
    if (M.n_cells) {
        uint32_t cell = (gidx / P.replicas_per_cell) % M.n_cells;
        rate = M.cell_d0[(size_t)cell * M.n_entities + M.src_id];
        mean = M.cell_d0[(size_t)cell * M.n_entities + M.srv_id];
        c_rt = M.cell_i0[(size_t)cell * M.n_entities + M.srv_id];
    }
    const double lambda = HS_DIV(1.0, mean);             /* exponential.py:36 */
    /* reciprocals for hs_div_by: exact x / rate and x / lambda in three fp64 instructions (0.0 = general division) */
    const double rate_recip = hs_recip_divisor_ok(rate) ? HS_DIV(1.0, rate) : 0.0;
    const double lambda_recip = hs_recip_divisor_ok(lambda) ? HS_DIV(1.0, lambda) : 0.0;
    hs_profile_desc prof_local;
    if (FLAGS & HS_LF_PROFILE) prof_local = M.prof;
    const hs_profile_desc *profp = (FLAGS & HS_LF_PROFILE) ? &prof_local : nullptr;
    constexpr bool SIMPLE = (FLAGS & HS_LF_SIMPLE) != 0;
    const bool poisson = SIMPLE ? true : (M.arr_kind == HS_ARR_POISSON);
    const bool expo = SIMPLE ? true : (M.svc_kind == HS_SVC_EXPONENTIAL);
    const bool lifo = SIMPLE ? false : (M.policy == HS_Q_LIFO);
    const int64_t cap = SIMPLE ? -1 : M.capacity;
    const int64_t stop_after = SIMPLE ? -1 : M.stop_after;
    const int32_t c_limit = SIMPLE ? 1 : c_rt;           /* FixedConcurrency._max_concurrent */
    hs_cont *heap = conts + (size_t)r * (uint32_t)M.c_max;   /* continuations beyond the earliest one */
    const bool dst_is_sink = SIMPLE ? true : (M.dst_kind == HS_ENT_SINK);
    const bool has_dst = SIMPLE ? true : (M.dst_id >= 0);
    const double *trace_arr = SIMPLE ? nullptr : P.trace_arr;
    const double *trace_svc = SIMPLE ? nullptr : P.trace_svc;
    const int dst_ev = dst_is_sink ? HS_EV_REQ_SINK : HS_EV_REQ_COUNTER;
    const uint32_t ring_mask = P.ring - 1u;
    hs_ring_entry *ring = rings + (size_t)r * P.ring;
    const bool windowed = (P.window_end_ns >= 0 && P.window_end_ns < P.end_ns);

    hs_event_record *rec = (FLAGS & HS_LF_REC) && O.records ? O.records + (size_t)r * P.record_cap : nullptr;
    hs_sink_sample *smp = (FLAGS & HS_LF_REC) && O.samples ? O.samples + (size_t)r * P.sample_cap : nullptr;
    double *svc_out = (FLAGS & HS_LF_REC) && O.service ? O.service + (size_t)r * P.service_cap : nullptr;
    uint32_t *hist = O.hist ? O.hist + (size_t)r * HS_HIST_BINS : nullptr;

    /* ---- replica state (registers; nowq in local memory, cold) ---------- */
    int64_t now, processed, tT, tC, c_created;
    uint64_t ctr, hash, iT, iC, arr_draws;
    int64_t dropped, n_svc;
    double svc_s, total_service, sum, comp, sumsq, mn, mx;
    uint32_t q_head, q_len, status, rec_pos, smp_pos, svc_pos;
    int32_t active, now_n;
    /* The item the next POLL delivers lives in this lane's 16-byte shared-memory slot
     * sh_head[tid].  After a pop the new head is fetched from the ring with cp.async
     * (LDGSTS: global -> shared, no destination register), i.e. a whole service time before
     * the next pop reads it, so no instruction waits on the ring's L2/HBM latency. */
    hs_ring_entry *const my_head = &sh_head[tid];
    const uint32_t my_head_s = (uint32_t)__cvta_generic_to_shared(my_head);
    /* recorder staging cursors: st_wr staged, st_fl flushed; rec_pos = ring slot of record st_fl */
    const bool staged = (FLAGS & HS_LF_REC) && O.records && P.record_cap >= 2 * HS_FLUSH && (P.record_cap % HS_FLUSH) == 0;
    uint32_t st_wr = 0, st_fl = 0;
    /* Sink samples: smp_sync <=> every earlier entry of the 64-byte group being filled is staged; smp_full <=> a
     * whole group is staged and waits for the next flush (its ring slots end at smp_pos) */
    const bool smp_groups = (FLAGS & HS_LF_REC) && smp && (P.sample_cap % HS_SMP_GROUP) == 0;
    bool smp_sync = false, smp_full = false;
    /* Service times in 64-byte chunks, written by the refill round as the draw buffer completes one (see
     * HS_REFILL_ROUND); other capacities are written entry by entry at the service start */
    const bool svc_chunks = (FLAGS & HS_LF_REC) && svc_out && (P.service_cap % HS_SVC_CHUNK) == 0;
    hs_now_ev nowq[HS_NOW_CAP];
    /* the Sink's current time bucket (HS_LF_BUCKETS; an empty type otherwise): stored when it moves on and at the end */
    typename hs_bucket_acc_of<(FLAGS & HS_LF_BUCKETS) != 0>::type bacc;
    if (FLAGS & HS_LF_BUCKETS) hs_bucket_reset(bacc);

    hs_lane_state *S = states + r;
    bool finished = !valid;
    if (P.resume) {
        if (S->done) finished = true;
        now = S->now; ctr = S->ctr; processed = S->processed; hash = S->hash;
        tT = S->tT; iT = S->iT; arr_draws = S->arr_draws;
        tC = S->tC; iC = S->iC; svc_s = S->svc_s; c_created = S->c_created;
        n_svc = S->n_svc; dropped = S->dropped;
        total_service = S->total_service;
        sum = S->sum; comp = S->comp; sumsq = S->sumsq; mn = S->mn; mx = S->mx;
        q_head = S->q_head; q_len = S->q_len; active = S->active; status = S->status;
        now_n = S->now_n;
        rec_pos = S->rec_pos; smp_pos = S->smp_pos; svc_pos = S->svc_pos;
        for (int i = 0; i < HS_NOW_CAP; ++i) nowq[i] = S->nowq[i];
        if (q_len > 0) *my_head = ring[(lifo ? q_head + q_len - 1 : q_head) & ring_mask];
    } else {
        now = 0; processed = 0; hash = HS_HASH_INIT; ctr = 0;
        arr_draws = 0; n_svc = 0;
        tT = 0; iT = 0; tC = 0; iC = 0; svc_s = 0.0; c_created = 0;
        dropped = 0;
        total_service = 0.0; sum = 0.0; comp = 0.0; sumsq = 0.0;
        mn = __longlong_as_double(0x7ff0000000000000LL); mx = __longlong_as_double(0xfff0000000000000LL);
        q_head = 0; q_len = 0; active = 0; status = 0; now_n = 0;
        rec_pos = 0; smp_pos = 0; svc_pos = 0;
        if (valid) { S->rejected = 0; S->skipped = 0; }   /* cold counters, kept in the state block */
        for (int i = 0; i < HS_NOW_CAP; ++i) { nowq[i].idx = 0; nowq[i].created = 0; nowq[i].payload_idx = 0; nowq[i].kind = 0; nowq[i].pad = 0; }
    }
    /* Generation cursors.  a_gen = arrival draws generated so far and t_gen = A_{a_gen}, the
     * provider's current_time after them; the pending SourceEvent is A_{arr_draws} = tT.
     * s_gen = service draws generated; service start number n_svc consumes draw n_svc.
     * After a pause the cursors restart at the consumed positions (a half-used Philox pair
     * is regenerated and its first half skipped).  With service chunks the service cursor restarts
     * at the start of the chunk n_svc lies in: the draws before n_svc are regenerated so that the
     * chunk's refill finds all of it in the buffer, and rewrites the ring slots of those draws with
     * the values an earlier launch put there; so s_gen - n_svc is negative until the first fill. */
    uint64_t a_gen = arr_draws, s_gen = svc_chunks ? (uint64_t)n_svc & ~(uint64_t)(HS_SVC_CHUNK - 1) : (uint64_t)n_svc;
    int64_t t_gen = P.resume ? tT : 0;

    /* next arrival time from t (arrival_time_provider.py:66-82); a result < t would be
     * popped and skipped as "time travel" by the loop (simulation.py:479-489), after which the
     * Source never ticks again: INT64_MAX marks that dead source. */
#define HS_NEXT_ARRIVAL(T, TARGET) hs_lane_next_arrival<(FLAGS & HS_LF_PROFILE) != 0>((T), (TARGET), rate, rate_recip, profp)

    /* one converged refill round: each lane that has room generates the next Philox
     * pair of each stream and stores the precomputed draws */
#define HS_REFILL_ROUND()                                                                    \
    do {                                                                                     \
        if (!finished && (uint32_t)(a_gen - arr_draws) + 2u <= ARR_BUF) {                    \
            double u0_ = 0.0, u1_ = 0.0, g0_ = 1.0, g1_ = 1.0;                               \
            if (poisson && !trace_arr) { hs_uniform_pair(seed, rid, sid_arr, a_gen >> 1, &u0_, &u1_); \
                                           g0_ = hs_exp1(u0_); g1_ = hs_exp1(u1_); }         \
            if (poisson && trace_arr) {                                                    \
                const uint64_t k_ = a_gen & ~1ull;                                           \
                if (k_ + 1 >= P.n_trace_arr) { status |= HS_ST_TRACE_EXHAUSTED; finished = true; } \
                else { g0_ = trace_arr[(size_t)r * P.n_trace_arr + k_]; g1_ = trace_arr[(size_t)r * P.n_trace_arr + k_ + 1]; } \
            }                                                                                \
            if (!(a_gen & 1)) {                                                              \
                t_gen = HS_NEXT_ARRIVAL(t_gen, g0_); a_gen++;                                \
                sh_t[a_gen % ARR_BUF][tid] = t_gen;                                          \
            }                                                                                \
            t_gen = HS_NEXT_ARRIVAL(t_gen, g1_); a_gen++;                                    \
            sh_t[a_gen % ARR_BUF][tid] = t_gen;                                              \
        }                                                                                    \
        bool chunk_ = false;                                                                 \
        if (!finished && (int32_t)(uint32_t)(s_gen - (uint64_t)n_svc) + 2 <= (int32_t)HS_DRAW_BUF) {   \
            double u0_ = 0.0, u1_ = 0.0;                                                     \
            int64_t d0_ = hs_seconds_to_ns(mean), d1_ = d0_;                                 \
            if (expo && !trace_svc) { hs_uniform_pair(seed, rid, sid_svc, s_gen >> 1, &u0_, &u1_); \
                                        d0_ = hs_exp_latency_ns_r(u0_, lambda, lambda_recip); d1_ = hs_exp_latency_ns_r(u1_, lambda, lambda_recip); } \
            if (expo && trace_svc) {       /* Duration.from_seconds(-log(1-U) / lambda)         */ \
                const uint64_t k_ = s_gen & ~1ull;                                           \
                if (k_ + 1 >= P.n_trace_svc) { status |= HS_ST_TRACE_EXHAUSTED; finished = true; } \
                else { d0_ = hs_seconds_to_ns(hs_div_by(trace_svc[(size_t)r * P.n_trace_svc + k_], lambda, lambda_recip));  \
                       d1_ = hs_seconds_to_ns(hs_div_by(trace_svc[(size_t)r * P.n_trace_svc + k_ + 1], lambda, lambda_recip)); } \
            }                                                                                \
            if (!(s_gen & 1)) {                                                              \
                const double s0_ = hs_ns_to_seconds(d0_);                                    \
                sh_svc[s_gen % HS_DRAW_BUF][tid] = s0_;                                      \
                s_gen++;                                                                     \
            }                                                                                \
            const double s1_ = hs_ns_to_seconds(d1_);                                        \
            sh_svc[s_gen % HS_DRAW_BUF][tid] = s1_;                                          \
            s_gen++;                                                                         \
            chunk_ = svc_chunks && (s_gen % HS_SVC_CHUNK) < 2u;   /* draws s_gen - 8 .. s_gen - 1 complete */ \
        }                                                                                    \
        if (FLAGS & HS_LF_REC) HS_SVC_FLUSH(chunk_);                                         \
    } while (0)

    /* The completed service chunks of the warp, written together: lane l moves draws 2 (l / 8), 2 (l / 8) + 1 of
     * the chunk of the (l % 8)-th owner, 8 chunks per store instruction.  The chunk is the owner's whole sh_svc
     * column, written in this round, so __syncwarp() orders those writes before the reads here (and the reads
     * before the next round's writes).  Its ring slot follows from svc_pos = n_svc mod service_cap: the chunk
     * starts 0..7 draws before n_svc.  Slots of draws not consumed yet are written ahead; the end of the
     * launch puts back what they held. */
#define HS_SVC_FLUSH(READY)                                                                  \
    do {                                                                                     \
        __syncwarp();                                                                        \
        uint32_t owners_ = __ballot_sync(0xffffffffu, (READY));                              \
        if (owners_) {                                                                       \
            uint32_t lane_;                                                                  \
            asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane_));                             \
            const uint32_t k_ = lane_ & 7u, pc_ = lane_ >> 3;                                \
            const uint32_t warp_r0_ = blockIdx.x * HS_LANE_THREADS + tid - lane_;            \
            const uint32_t back_ = (uint32_t)((uint64_t)n_svc - (s_gen - HS_SVC_CHUNK));     \
            const uint32_t my_slot_ = svc_pos >= back_ ? svc_pos - back_ : svc_pos + P.service_cap - back_; \
            do {                                                                             \
                const uint32_t owner_ = hs_kth_set_lane<8>(owners_, k_);                     \
                uint32_t rest_ = owners_;                                                    \
                _Pragma("unroll") for (uint32_t q_ = 0; q_ < 8; ++q_) rest_ &= rest_ - 1u;    \
                const uint32_t o_slot_ = __shfl_sync(0xffffffffu, my_slot_, owner_ < 32u ? owner_ : lane_); \
                if (owner_ < 32u) {                                                          \
                    const uint32_t col_ = tid - lane_ + owner_;                              \
                    const uint64_t a_ = (uint64_t)__double_as_longlong(sh_svc[2u * pc_][col_]);      \
                    const uint64_t b_ = (uint64_t)__double_as_longlong(sh_svc[2u * pc_ + 1u][col_]); \
                    __stcs((uint4 *)(O.service + (size_t)(warp_r0_ + owner_) * P.service_cap + o_slot_) + pc_, \
                           make_uint4((uint32_t)a_, (uint32_t)(a_ >> 32), (uint32_t)b_, (uint32_t)(b_ >> 32))); \
                }                                                                            \
                owners_ = rest_;                                                             \
            } while (owners_);                                                               \
            __syncwarp();                                                                    \
        }                                                                                    \
    } while (0)

    /* Sink sample into its ring: staged in the lane's shared-memory column until its 64-byte group is full,
     * which the next loop top writes out (the fourth sample in the free record-staging row, see sh_rec).  A
     * group that was begun before this launch (resume inside a group) or rings whose capacity is not a
     * multiple of the group are written entry by entry. */
#define HS_SMP_STORE(W)                                                                      \
    do {                                                                                     \
        const uint32_t p_ = smp_pos, q_ = p_ % HS_SMP_GROUP;                                 \
        if (q_ == 0u) smp_sync = smp_groups;                                                 \
        if (smp_sync) {                                                                      \
            uint4 *d_ = (q_ < HS_SMP_GROUP - 1) ? &sh_smp[q_][tid] : &sh_rec[(st_fl + HS_STAGE - 1u) % HS_STAGE][tid]; \
            *d_ = (W);                                                                       \
            smp_full = (q_ == HS_SMP_GROUP - 1);                                             \
        } else *(uint4 *)(smp + p_) = (W);                                                   \
        smp_pos = (p_ + 1 == P.sample_cap) ? 0u : p_ + 1;                                    \
    } while (0)
    /* service time at its start: written here only when the ring does not take whole chunks */
#define HS_SVC_STORE(V)                                                                      \
    do {                                                                                     \
        if (!svc_chunks) svc_out[svc_pos] = (V);                                             \
        svc_pos = (svc_pos + 1 == P.service_cap) ? 0u : svc_pos + 1;                         \
    } while (0)

#define HS_RECORD(KIND, IDX, ENT)                                                            \
    do {                                                                                     \
        if (FLAGS & HS_LF_HASH) hash = hs_hash_step(hash, now, hs_record_word1((IDX), (KIND), (uint32_t)(ENT))); \
        if ((FLAGS & HS_LF_REC) && rec) {                                                    \
            uint4 w_;                                                                        \
            w_.x = (uint32_t)(uint64_t)now; w_.y = (uint32_t)((uint64_t)now >> 32);          \
            w_.z = (uint32_t)(IDX); w_.w = (uint32_t)(KIND) | ((uint32_t)(ENT) << 16);       \
            /* staging non-empty implies rec_pos is group aligned (it then only moves by whole groups) */ \
            if (staged && (st_wr != st_fl || (rec_pos % HS_FLUSH) == 0)) { sh_rec[st_wr % HS_STAGE][tid] = w_; st_wr++; } \
            else { __stcs((uint4 *)(rec + rec_pos), w_);                                     \
                   rec_pos = (rec_pos + 1 == P.record_cap) ? 0u : rec_pos + 1; }             \
        }                                                                                    \
    } while (0)
#define HS_EMIT(KIND, IDX, ENT) do { HS_RECORD(KIND, IDX, ENT); processed++; } while (0)

    /* Source.handle_event's arrival part: the next SourceEvent (source.py:166-170) */
#define HS_NEXT_TICK()                                                                       \
    do { arr_draws++; tT = sh_t[arr_draws % ARR_BUF][tid];                                   \
         if (tT == HS_T_EXHAUSTED) tT = INT64_MAX; else iT = ctr++; } while (0)

    /* Server.handle_queued_event up to its yield, for the payload (CREATED):
     * inline ProcessContinuation index, acquire (the caller has checked
     * active < c_limit), sample, schedule resume
     * (server.py:217-253, event.py:314-325,499-508).                            */
#define HS_SERVICE_START(CREATED)                                                            \
    do {                                                                                     \
        const uint32_t k_ = (uint32_t)((uint64_t)n_svc % HS_DRAW_BUF);                       \
        const int64_t delta_ = hs_seconds_to_ns(sh_svc[k_][tid]);   /* event.py:499, temporal.py:221 */ \
        if ((FLAGS & HS_LF_REC) && svc_out) HS_SVC_STORE(sh_svc[k_][tid]);                     \
        n_svc++;                                                                             \
        { const double sv_ = sh_svc[k_][tid]; const uint64_t i_ = ctr + 1; ctr += 2;         \
          HS_C_PUSH(now + delta_, i_, (CREATED), sv_); }                                     \
    } while (0)

#define HS_SINK(CREATED)                                                                     \
    do {                                                                                     \
        if (dst_is_sink) {                                                                   \
            const double lat_ = hs_ns_to_seconds(now - (CREATED));                           \
            if (hist) atomicAdd(hist + hs_latency_bin(now - (CREATED)), 1u);  /* RED: no return value, no stall */ \
            hs_neumaier_add(&sum, &comp, lat_); sumsq = HS_ADD(sumsq, HS_MUL(lat_, lat_));   \
            if (lat_ < mn) mn = lat_;                                                        \
            if (lat_ > mx) mx = lat_;                                                        \
            if (FLAGS & HS_LF_BUCKETS) hs_bucket_add(BK, r, 0u, bacc, now, lat_);          \
            if ((FLAGS & HS_LF_REC) && smp) {                                                \
                uint4 w_; const uint64_t lb_ = (uint64_t)__double_as_longlong(lat_);         \
                w_.x = (uint32_t)(uint64_t)now; w_.y = (uint32_t)((uint64_t)now >> 32);      \
                w_.z = (uint32_t)lb_; w_.w = (uint32_t)(lb_ >> 32);                          \
                HS_SMP_STORE(w_); }                                                          \
        }                                                                                    \
    } while (0)

    /* FIFOQueue / LIFOQueue (queue_policy.py:75-156) on the HBM ring + the register copy
     * of the next item to be delivered */
#define HS_Q_PUSH(CREATED, IDX)                                                              \
    do {                                                                                     \
        hs_ring_entry e_; e_.created = (CREATED); e_.idx = (IDX);                            \
        ring[(q_head + q_len) & ring_mask] = e_;                                             \
        if (lifo) { asm volatile("cp.async.wait_group 0;" ::: "memory"); *my_head = e_; }    \
        else if (q_len == 0) *my_head = e_;                                                  \
        q_len++;                                                                             \
    } while (0)
#define HS_Q_POP(CREATED, IDX)                                                               \
    do {                                                                                     \
        asm volatile("cp.async.wait_group 0;" ::: "memory");                                 \
        { const hs_ring_entry h_ = *my_head; (CREATED) = h_.created; (IDX) = h_.idx; }       \
        if (!lifo) q_head++;                                                                 \
        q_len--;                                                                             \
        if (q_len == 0) q_head = 0;   /* an empty queue restarts at slot 0: the rings' hot lines stay in L2 */ \
        if (q_len > 0) {                                                                     \
            const hs_ring_entry *n_ = ring + ((lifo ? q_head + q_len - 1 : q_head) & ring_mask); \
            asm volatile("cp.async.ca.shared.global [%0], [%1], 16;\n\tcp.async.commit_group;" \
                         :: "r"(my_head_s), "l"(n_) : "memory");                             \
        }                                                                                    \
    } while (0)

    /* The set of pending continuations: the minimum (time, sort_index) lives in the registers
     * tC/iC/c_created/svc_s, the other (active - 1) in a binary min-heap in HBM. */
#define HS_CLT(T1, I1, T2, I2) ((T1) < (T2) || ((T1) == (T2) && (I1) < (I2)))
#define HS_C_PUSH(T, I, CR, SV)                                                              \
    do {                                                                                     \
        if (active == 0) { tC = (T); iC = (I); c_created = (CR); svc_s = (SV); }             \
        else {                                                                               \
            hs_cont n_;                                                                      \
            if (HS_CLT((T), (I), tC, iC)) { n_.t = tC; n_.idx = iC; n_.created = c_created; n_.svc_s = svc_s; \
                                            tC = (T); iC = (I); c_created = (CR); svc_s = (SV); } \
            else { n_.t = (T); n_.idx = (I); n_.created = (CR); n_.svc_s = (SV); }           \
            int k_ = active - 1;                       /* sift up */                         \
            while (k_ > 0) { const int p_ = (k_ - 1) >> 1; const hs_cont q_ = heap[p_];      \
                             if (!HS_CLT(n_.t, n_.idx, q_.t, q_.idx)) break; heap[k_] = q_; k_ = p_; } \
            heap[k_] = n_;                                                                   \
        }                                                                                    \
        active++;                                                                            \
    } while (0)
    /* remove the earliest continuation (the registers) and promote the heap's minimum */
#define HS_C_POP()                                                                           \
    do {                                                                                     \
        active = active > 0 ? active - 1 : 0;          /* FixedConcurrency.release */        \
        if (active > 0) {                                                                    \
            const hs_cont top_ = heap[0];                                                    \
            tC = top_.t; iC = top_.idx; c_created = top_.created; svc_s = top_.svc_s;        \
            const int n2_ = active - 1;                /* elements left in the heap */       \
            if (n2_ > 0) { const hs_cont last_ = heap[n2_]; int k_ = 0;                      \
                while (true) { int ch_ = 2 * k_ + 1; if (ch_ >= n2_) break;                  \
                    hs_cont a_ = heap[ch_];                                                  \
                    if (ch_ + 1 < n2_) { const hs_cont b_ = heap[ch_ + 1]; if (HS_CLT(b_.t, b_.idx, a_.t, a_.idx)) { a_ = b_; ch_++; } } \
                    if (!HS_CLT(a_.t, a_.idx, last_.t, last_.idx)) break; heap[k_] = a_; k_ = ch_; } \
                heap[k_] = last_; }                                                          \
        }                                                                                    \
    } while (0)

#define HS_PUSH_NOW(KIND, IDX, CREATED, PIDX)                                                \
    do {                                                                                     \
        if (now_n >= HS_NOW_CAP) { status |= HS_ST_FEL_OVERFLOW; }                           \
        else { nowq[now_n].idx = (IDX); nowq[now_n].created = (CREATED); nowq[now_n].payload_idx = (PIDX); \
               nowq[now_n].kind = (KIND); now_n++; }                                         \
    } while (0)

    /* ---- fill the draw buffers, then bootstrap --------------------------- */
#pragma unroll 1
    for (int k = 0; k < HS_DRAW_BUF / 2; ++k) HS_REFILL_ROUND();
    if (!P.resume && !finished) {
        /* Simulation.__init__: source.start() draws the first arrival and the
         * SourceEvent takes index 0 of the GLOBAL counter (simulation.py:77,145-154);
         * run() then restarts the per-heap counter at 0 (event_heap.py:48).        */
        arr_draws = 1; tT = sh_t[1][tid];
        if (tT == HS_T_EXHAUSTED) tT = INT64_MAX;      /* source.start(): RuntimeError, no first tick */
        iT = 0; ctr = 0;
    }

    const uint32_t stop_bits = HS_ST_QUEUE_OVERFLOW | HS_ST_FEL_OVERFLOW;
    /* SIMPLE kernels: conditions that only a generic step can change, folded into one flag
     * (a stop bit is set; recorder staging not yet group aligned after a resume) */
#define HS_STICKY_SLOW() (((status & stop_bits) != 0) || ((FLAGS & HS_LF_REC) && rec && !(staged && (st_wr != st_fl || (rec_pos % HS_FLUSH) == 0))))
    bool sticky_slow = HS_STICKY_SLOW();
    const int64_t ev_fast_limit = P.max_events - 8;     /* a chain is <= 6 events: single-step near the limit */
    const int64_t fast_limit = (windowed && P.window_end_ns < P.end_ns) ? P.window_end_ns : P.end_ns;
    bool paused = false;
    while (true) {
        /* converged top of the loop: vote on termination and on refilling */
        const bool need = !finished && (a_gen == arr_draws || s_gen == (uint64_t)n_svc);
        const unsigned todo = __ballot_sync(0xffffffffu, !finished);
        if (todo == 0u) break;
        if (__any_sync(0xffffffffu, need)) HS_REFILL_ROUND();
        /* Lanes read each other's staging here: the __syncwarp()s order the owners' earlier staging writes before
         * these reads, and these reads before the owners' next staging writes. */
        if (FLAGS & HS_LF_REC) __syncwarp();
        if (FLAGS & HS_LF_REC) {
            /* the full 64-byte Sink-sample groups of the warp, eight per store instruction: lane l moves sample l / 8
             * of the group of the (l % 8)-th owner.  Before the record flush, which moves st_fl and with it the
             * row that holds the fourth sample. */
            uint32_t owners = __ballot_sync(0xffffffffu, smp_full);
            if (owners) {
                uint32_t lane;
                asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
                const uint32_t k = lane & 7u, pc = lane >> 3;
                const uint32_t warp_r0 = blockIdx.x * HS_LANE_THREADS + tid - lane;
                const uint32_t my_slot = (smp_pos == 0u ? P.sample_cap : smp_pos) - HS_SMP_GROUP;
                do {
                    const uint32_t owner = hs_kth_set_lane<8>(owners, k);
                    uint32_t rest = owners;
#pragma unroll
                    for (uint32_t q = 0; q < 8; ++q) rest &= rest - 1u;
                    const uint32_t src = owner < 32u ? owner : lane;
                    const uint32_t o_slot = __shfl_sync(0xffffffffu, my_slot, src);
                    const uint32_t o_row = (__shfl_sync(0xffffffffu, st_fl, src) + HS_STAGE - 1u) % HS_STAGE;
                    if (owner < 32u) {
                        const uint32_t col = tid - lane + owner;
                        __stcs((uint4 *)(O.samples + (size_t)(warp_r0 + owner) * P.sample_cap + o_slot + pc),
                               pc < HS_SMP_GROUP - 1 ? sh_smp[pc][col] : sh_rec[o_row][col]);
                    }
                    owners = rest;
                } while (owners);
                __syncwarp();
                smp_full = false;
            }
        }
        if ((FLAGS & HS_LF_REC) && staged) {
            /* the warp writes the full 128-byte groups of all its lanes together, four whole lines per store
             * instruction: lane l moves record l / 4 of the group of the (l % 4)-th owner of the round (so a
             * quarter-warp reads two rows of four staging columns).  An owner's group is rows 0-7 or 8-15 of
             * its column, since st_fl is a multiple of 8; its ring slot rec_pos is group aligned. */
            const bool full = (st_wr - st_fl) >= HS_FLUSH;
            uint32_t owners = __ballot_sync(0xffffffffu, full);
            if (owners) {
                /* everything below is derived from the lane index read here, so none of it is hoisted out
                 * of the event loop, where registers are scarce; the owner's ring is found from the kernel
                 * parameters, so only two 32-bit values cross lanes */
                uint32_t lane;
                asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
                const uint32_t k = lane & 3u, row = lane >> 2;
                const uint32_t warp_r0 = blockIdx.x * HS_LANE_THREADS + tid - lane;   /* replica of lane 0 */
                do {
                    /* the k-th lowest owner left (32: none) */
                    const uint32_t owner = hs_kth_set_lane<4>(owners, k);
                    uint32_t rest = owners;
#pragma unroll
                    for (uint32_t q = 0; q < 4; ++q) rest &= rest - 1u;
                    const uint32_t src = owner < 32u ? owner : lane;
                    const uint32_t o_pos = __shfl_sync(0xffffffffu, rec_pos, src);
                    const uint32_t o_row = __shfl_sync(0xffffffffu, st_fl, src) % HS_STAGE + row;
                    if (owner < 32u)
                        __stcs((uint4 *)(O.records + (size_t)(warp_r0 + owner) * P.record_cap + o_pos + row),
                               sh_rec[o_row][tid - lane + owner]);
                    owners = rest;
                } while (owners);
                __syncwarp();
                if (full) { st_fl += HS_FLUSH; rec_pos = (rec_pos + HS_FLUSH == P.record_cap) ? 0u : rec_pos + HS_FLUSH; }
            }
        }
        /* SIMPLE: the three shared-memory operands of the next chain, requested before any of them is used:
         * next arrival time, next service time, queue head */
        int64_t tT_next = 0; double sv_next = 0.0; hs_ring_entry h; h.created = 0; h.idx = 0;
        if (SIMPLE) {
            tT_next = sh_t[(arr_draws + 1) % ARR_BUF][tid];
            sv_next = sh_svc[(uint32_t)((uint64_t)n_svc % HS_DRAW_BUF)][tid];
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            h = *my_head;                                    /* next queued request (meaningful if q_len > 0) */
        }
        if (finished) continue;

        if (SIMPLE && now_n == 0) {
            /* ===== M/M/1 shape (HS_LF_SIMPLE): one converged, branch-free chain per iteration =====
             * Both chains -- arrival TICK -> ENQUEUE [-> NOTIFY [-> POLL -> DELIVER -> WORKER]] and completion
             * CONTINUATION -> SINK -> POLL [-> DELIVER -> WORKER] -- are the same straight-line code with
             * per-lane selects, so the lanes of a warp never split by chain.  Everything that could make the
             * events created at `now` NOT the next pops is tested up front, before any state changes; such a
             * lane takes the generic one-event step below instead:
             *   a tie between the pending tick and the continuation, a next tick that is not later than this one
             *   (zero inter-arrival) or does not exist, the run / window end, a stop bit, the event limit, a
             *   full device ring, and recorder staging that is not group aligned yet (first events after a resume). */
            const bool busy = active > 0;
            const bool pickC = busy && tC < tT;
            const bool isA = !pickC;
            const int64_t tn = pickC ? tC : tT;
            /* (tn >= now always holds here: arrival times are generated non-decreasing -- an earlier one is
             * stored as INT64_MAX, "time travel" -- and a continuation resumes at now + delta, delta >= 0) */
            bool slow = sticky_slow || (busy && tC == tT) || (tn > fast_limit) || (processed > ev_fast_limit) ||
                        (isA && tT_next <= tn) || (q_len >= P.ring);
            if (FLAGS & HS_LF_PROFILE) slow = slow || (isA && tT_next == HS_T_EXHAUSTED);
            if (!slow) {
                now = tn;
                const bool q_empty = (q_len == 0);
                const bool start = isA ? (q_empty && !busy) : !q_empty;      /* a service starts in this chain */
                const uint64_t c0 = ctr;
                const uint64_t idx0 = isA ? iT : iC;
                const uint64_t widx = isA ? c0 : h.idx;                      /* the payload WORKER carries */
                const int64_t start_created = isA ? now : h.created;
                const uint32_t nrec = isA ? (2u + (q_empty ? 1u : 0u) + (start ? 3u : 0u)) : (3u + (start ? 2u : 0u));
                ctr = c0 + (isA ? (2u + (q_empty ? 1u : 0u) + (start ? 4u : 0u)) : (2u + (start ? 3u : 0u)));
                processed += nrec;
                if ((FLAGS & HS_LF_HASH) || ((FLAGS & HS_LF_REC) && rec)) {
                    /* slot:   0            1        2             3              4               5
                     * A:      TICK iT      ENQ c0   NOTIFY c0+2   POLL c0+3      DELIVER c0+4    WORKER c0
                     * C:      CONT iC      SINK c0  POLL c0+1     DELIVER c0+2   WORKER item     -        */
                    const uint32_t esrv = (uint32_t)M.srv_id << 16;
                    uint32_t z[6], w[6]; bool v[6];
                    z[0] = (uint32_t)idx0; z[1] = (uint32_t)c0; z[2] = (uint32_t)c0 + (isA ? 2u : 1u);
                    z[3] = (uint32_t)c0 + (isA ? 3u : 2u); z[4] = isA ? (uint32_t)c0 + 4u : (uint32_t)widx; z[5] = (uint32_t)c0;
                    w[0] = isA ? ((uint32_t)HS_EV_SOURCE_TICK | ((uint32_t)M.src_id << 16)) : ((uint32_t)HS_EV_CONTINUATION | esrv);
                    w[1] = isA ? ((uint32_t)HS_EV_REQ_ENQUEUE | esrv) : ((uint32_t)HS_EV_REQ_SINK | ((uint32_t)M.dst_id << 16));
                    w[2] = (isA ? (uint32_t)HS_EV_NOTIFY : (uint32_t)HS_EV_POLL) | esrv;
                    w[3] = (isA ? (uint32_t)HS_EV_POLL : (uint32_t)HS_EV_DELIVER) | esrv;
                    w[4] = (isA ? (uint32_t)HS_EV_DELIVER : (uint32_t)HS_EV_REQ_WORKER) | esrv;
                    w[5] = (uint32_t)HS_EV_REQ_WORKER | esrv;
                    v[0] = true; v[1] = true; v[2] = isA ? q_empty : true; v[3] = start; v[4] = start; v[5] = isA && start;
                    const uint32_t nlo = (uint32_t)(uint64_t)now, nhi = (uint32_t)((uint64_t)now >> 32);
#pragma unroll
                    for (int j = 0; j < 6; ++j) {
                        if (v[j]) {
                            if (FLAGS & HS_LF_HASH) hash = hs_hash_step(hash, now, (uint64_t)z[j] | ((uint64_t)(w[j] & 0xffu) << 32) | ((uint64_t)(w[j] >> 16) << 40));
                            if ((FLAGS & HS_LF_REC) && rec) sh_rec[(st_wr + (uint32_t)j) % HS_STAGE][tid] = make_uint4(nlo, nhi, z[j], w[j]);
                        }
                    }
                    if ((FLAGS & HS_LF_REC) && rec) st_wr += nrec;
                }
                /* The updates as selects + predicated memory operations, not as one branch per chain: no branch, no
                 * reconvergence point, no register shuffling where the chains meet again.  Measured A/B against the
                 * two-branch form (tools/bench_lane.py), it won without the recorder and with the order hash.  With
                 * the recorder alone the two forms run at the same speed (within run-to-run spread,
                 * profiles/h100_rec_flush_ab.txt), but the two-branch form spills registers next to the warp-wide
                 * record flush (ptxas: 320 B stack, 64 B spill stores) and the predicated one does not. */
                const bool isC = !isA;
                /* Source: payload index c0, next SourceEvent index c0 + 1 (source.py:166-170) */
                arr_draws += isA ? 1ull : 0ull;
                tT = isA ? tT_next : tT;
                iT = isA ? c0 + 1 : iT;
                /* Server resumes after its yield, the Sink takes the request (server.py:255-273, common.py:36-44) */
                {
                    const double ts_ = HS_ADD(total_service, svc_s);
                    total_service = isC ? ts_ : total_service;
                    const int64_t dlat_ = now - c_created;
                    const double lat_ = hs_ns_to_seconds(dlat_);
                    if (isC && hist) atomicAdd(hist + hs_latency_bin(dlat_), 1u);
                    {   /* hs_neumaier_add, branch-free: c += (hi - t) + lo with (hi, lo) = (s, x) ordered by magnitude */
                        const double t_ = HS_ADD(sum, lat_);
                        const bool big_ = hs_fabs(sum) >= hs_fabs(lat_);
                        const double hi_ = big_ ? sum : lat_, lo_ = big_ ? lat_ : sum;
                        const double c2_ = HS_ADD(comp, HS_ADD(HS_SUB(hi_, t_), lo_));
                        sum = isC ? t_ : sum; comp = isC ? c2_ : comp;
                    }
                    const double q2_ = HS_ADD(sumsq, HS_MUL(lat_, lat_));
                    sumsq = isC ? q2_ : sumsq;
                    mn = (isC && lat_ < mn) ? lat_ : mn;
                    mx = (isC && lat_ > mx) ? lat_ : mx;
                    if (isC && (FLAGS & HS_LF_BUCKETS)) hs_bucket_add(BK, r, 0u, bacc, now, lat_);
                    if (isC && (FLAGS & HS_LF_REC) && smp) {
                        uint4 w_; const uint64_t lb_ = (uint64_t)__double_as_longlong(lat_);
                        w_.x = (uint32_t)(uint64_t)now; w_.y = (uint32_t)((uint64_t)now >> 32);
                        w_.z = (uint32_t)lb_; w_.w = (uint32_t)(lb_ >> 32);
                        HS_SMP_STORE(w_);
                    }
                }
                /* Queue: the request waits (arrival, no service start) / the head is delivered (completion with a start) */
                const bool do_push = isA && !start, do_pop = isC && start;
                if (do_push) {
                    hs_ring_entry e_; e_.created = now; e_.idx = c0;
                    ring[(q_head + q_len) & ring_mask] = e_;
                    if (q_empty) *my_head = e_;
                }
                q_len = q_len + (do_push ? 1u : 0u) - (do_pop ? 1u : 0u);
                q_head = do_pop ? (q_len == 0 ? 0u : q_head + 1u) : q_head;      /* an empty queue restarts at slot 0 */
                if (do_pop && q_len > 0) {
                    const hs_ring_entry *n_ = ring + (q_head & ring_mask);
                    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;\n\tcp.async.commit_group;"
                                 :: "r"(my_head_s), "l"(n_) : "memory");
                }
                /* Server.handle_queued_event up to its yield (server.py:217-253): the scheduled ProcessContinuation
                 * takes the last index of the chain */
                if (start && (FLAGS & HS_LF_REC) && svc_out) HS_SVC_STORE(sv_next);
                n_svc += start ? 1 : 0;
                tC = start ? now + hs_seconds_to_ns(sv_next) : tC;
                iC = start ? ctr - 1 : iC;
                c_created = start ? start_created : c_created;
                svc_s = start ? sv_next : svc_s;
                active = start ? 1 : (isA ? active : 0);
                continue;
            }
        }

        if (!SIMPLE && now_n == 0) {
            const bool pickC = active > 0 && (tC < tT || (tC == tT && iC < iT));
            const int64_t tn = pickC ? tC : tT;
            /* fast path <=> the chosen event is not tied, lies inside both the run and the window
             * (so `now <= end` holds before and after), and nothing exceptional is pending */
            const bool slow = (active > 0 && tC == tT) || (tn > fast_limit) || (tn < now) || (status & stop_bits) ||
                              (processed + 8 > P.max_events);   /* a chain is <= 6 events: single-step near the limit */
            if (!slow) {
                now = tn;
                /* Recorder kernels emit the chain's first event and the common tail DELIVER -> WORKER ->
                 * service start once for both chains, so that the lanes of both run that code together
                 * (+6 % in record mode); without the record stores the shared tail only adds a
                 * reconvergence point (-5 % in summary mode), so those kernels keep the chains apart. */
                constexpr bool MERGED = (FLAGS & HS_LF_REC) != 0;
                if (MERGED) HS_EMIT(pickC ? HS_EV_CONTINUATION : HS_EV_SOURCE_TICK, pickC ? iC : iT, pickC ? M.srv_id : M.src_id);
                bool start = false; int64_t start_created = 0; uint64_t worker_idx = 0;
                if (!pickC) {
                    /* ===== fused arrival chain ================================== */
                    if (!MERGED) HS_EMIT(HS_EV_SOURCE_TICK, iT, M.src_id);
                    const bool payload = !(stop_after >= 0 && now > stop_after);  /* source.py:68 */
                    uint64_t idxP = 0;
                    if (payload) idxP = ctr++; else S->skipped++;
                    HS_NEXT_TICK();
                    if (!payload) continue;
                    if (tT <= now) {          /* zero inter-arrival: the new tick ties with the chain */
                        HS_PUSH_NOW(HS_EV_REQ_ENQUEUE, idxP, now, 0);
                        continue;
                    }
                    /* Queue._handle_enqueue (queue.py:122-147) */
                    HS_EMIT(HS_EV_REQ_ENQUEUE, idxP, M.srv_id);
                    const bool was_empty = (q_len == 0);
                    if (cap >= 0 && (int64_t)q_len >= cap) { dropped++; continue; }
                    if (q_len >= P.ring) { status |= HS_ST_QUEUE_OVERFLOW; continue; }
                    if (!was_empty || active >= c_limit) {
                        /* request waits in the buffer */
                        HS_Q_PUSH(now, idxP);
                        if (was_empty) {      /* notify, but the worker is busy: no poll (queue_driver.py:92-96) */
                            uint64_t idxN = ctr++;
                            HS_EMIT(HS_EV_NOTIFY, idxN, M.srv_id);
                        }
                        continue;
                    }
                    /* buffer was empty and the worker is idle: NOTIFY -> POLL -> DELIVER -> WORKER;
                     * the item is pushed and popped again at once (FIFO and LIFO agree).          */
                    HS_RECORD(HS_EV_NOTIFY, ctr, M.srv_id);
                    HS_RECORD(HS_EV_POLL, ctr + 1, M.srv_id);
                    ctr += 2; processed += 2;
                    if (MERGED) { start = true; start_created = now; worker_idx = idxP; }
                    else {
                        HS_RECORD(HS_EV_DELIVER, ctr, M.srv_id);
                        HS_RECORD(HS_EV_REQ_WORKER, idxP, M.srv_id);
                        ctr += 1; processed += 2;
                        HS_SERVICE_START(now);
                        continue;
                    }
                } else {
                    /* ===== fused completion chain =============================== */
                    if (!MERGED) HS_EMIT(HS_EV_CONTINUATION, iC, M.srv_id);
                    total_service = HS_ADD(total_service, svc_s);
                    const int64_t done_created = c_created;
                    HS_C_POP();                                /* release + promote the next continuation */
                    uint64_t idxF = 0;
                    if (has_dst) idxF = ctr++;                 /* Entity.forward */
                    uint64_t idxPoll = 0; bool poll = (active < c_limit);
                    if (poll) idxPoll = ctr++;                 /* schedule_poll hook */
                    if (active > 0 && tC == now) {
                        /* another continuation resumes at this very nanosecond: its (older) index sorts
                         * before the events just created, so hand them to the generic path */
                        if (has_dst) HS_PUSH_NOW(dst_ev, idxF, done_created, 0);
                        if (poll) HS_PUSH_NOW(HS_EV_POLL, idxPoll, 0, 0);
                        continue;
                    }
                    if (has_dst) { HS_EMIT(dst_ev, idxF, M.dst_id); HS_SINK(done_created); }
                    if (!poll) continue;
                    HS_EMIT(HS_EV_POLL, idxPoll, M.srv_id);
                    if (q_len == 0) continue;                  /* Queue._handle_poll: empty */
                    uint64_t it_idx;
                    HS_Q_POP(start_created, it_idx);
                    if (MERGED) { start = true; worker_idx = it_idx; }
                    else {
                        HS_RECORD(HS_EV_DELIVER, ctr, M.srv_id);
                        HS_RECORD(HS_EV_REQ_WORKER, it_idx, M.srv_id);
                        ctr += 1; processed += 2;
                        HS_SERVICE_START(start_created);
                        continue;
                    }
                }
                if (MERGED && start) {
                    HS_RECORD(HS_EV_DELIVER, ctr, M.srv_id);
                    HS_RECORD(HS_EV_REQ_WORKER, worker_idx, M.srv_id);
                    ctr += 1; processed += 2;
                    HS_SERVICE_START(start_created);
                }
                continue;
            }
        }

        /* ===== generic single-event step (ties, run end, window end, leftovers) ========= */
        if (!(now <= P.end_ns)) { finished = true; continue; }                 /* simulation.py:472 */
        if (status & stop_bits) { finished = true; continue; }
        if (now_n == 0 && tT == INT64_MAX && active == 0) { finished = true; continue; }   /* heap exhausted */
        if (processed >= P.max_events) { status |= HS_ST_EVENT_LIMIT; finished = true; continue; }
        {
            /* pop the (time, sort_index) minimum of T, C and nowq (event.py:337-344) */
            int which = -1;                 /* -1 T, -2 C, >=0 nowq slot */
            int64_t bt = tT; uint64_t bi = iT;
            if (active > 0 && (tC < bt || (tC == bt && iC < bi))) { which = -2; bt = tC; bi = iC; }
            for (int i = 0; i < now_n; ++i) {
                if (now < bt || (now == bt && nowq[i].idx < bi)) { which = i; bt = now; bi = nowq[i].idx; }
            }
            if (windowed && bt > P.window_end_ns) { paused = true; finished = true; continue; }
            if (bt < now) {                 /* "time travel": popped and skipped, not processed
                                               (simulation.py:479-489); only a SourceEvent can do it */
                tT = INT64_MAX; continue;
            }
            int kind; int64_t e_created = 0; uint64_t e_pidx = 0;
            if (which == -1) kind = HS_EV_SOURCE_TICK;
            else if (which == -2) kind = HS_EV_CONTINUATION;
            else {
                kind = nowq[which].kind; e_created = nowq[which].created; e_pidx = nowq[which].payload_idx;
                now_n--; nowq[which] = nowq[now_n];
            }
            now = bt;
            switch (kind) {
            case HS_EV_SOURCE_TICK: {
                HS_EMIT(HS_EV_SOURCE_TICK, bi, M.src_id);
                const bool payload = !(stop_after >= 0 && now > stop_after);
                uint64_t idxP = 0;
                if (payload) idxP = ctr++; else S->skipped++;
                HS_NEXT_TICK();
                if (payload) HS_PUSH_NOW(HS_EV_REQ_ENQUEUE, idxP, now, 0);
                break;
            }
            case HS_EV_REQ_ENQUEUE: {
                HS_EMIT(HS_EV_REQ_ENQUEUE, bi, M.srv_id);
                const bool was_empty = (q_len == 0);
                if (cap >= 0 && (int64_t)q_len >= cap) { dropped++; break; }
                if (q_len >= P.ring) { status |= HS_ST_QUEUE_OVERFLOW; break; }
                HS_Q_PUSH(e_created, bi);
                if (was_empty) { uint64_t i_ = ctr++; HS_PUSH_NOW(HS_EV_NOTIFY, i_, 0, 0); }
                break;
            }
            case HS_EV_NOTIFY:
                HS_EMIT(HS_EV_NOTIFY, bi, M.srv_id);
                if (active < c_limit) { uint64_t i_ = ctr++; HS_PUSH_NOW(HS_EV_POLL, i_, 0, 0); }
                break;
            case HS_EV_POLL:
                HS_EMIT(HS_EV_POLL, bi, M.srv_id);
                if (q_len > 0) {
                    int64_t it_created; uint64_t it_idx;
                    HS_Q_POP(it_created, it_idx);
                    uint64_t i_ = ctr++;
                    HS_PUSH_NOW(HS_EV_DELIVER, i_, it_created, it_idx);
                }
                break;
            case HS_EV_DELIVER:
                HS_EMIT(HS_EV_DELIVER, bi, M.srv_id);
                HS_PUSH_NOW(HS_EV_REQ_WORKER, e_pidx, e_created, 0);   /* payload keeps its old index */
                break;
            case HS_EV_REQ_WORKER:
                HS_EMIT(HS_EV_REQ_WORKER, bi, M.srv_id);
                if (active >= c_limit) {    /* acquire failed (server.py:223-234): hooks still run */
                    ctr++; S->rejected++; status |= HS_ST_REJECT_PATH;
                    if (active < c_limit) { uint64_t i_ = ctr++; HS_PUSH_NOW(HS_EV_POLL, i_, 0, 0); }
                } else {
                    HS_SERVICE_START(e_created);
                }
                break;
            case HS_EV_CONTINUATION: {
                HS_EMIT(HS_EV_CONTINUATION, bi, M.srv_id);
                total_service = HS_ADD(total_service, svc_s);
                const int64_t done_created = c_created;
                HS_C_POP();
                if (has_dst) { uint64_t i_ = ctr++; HS_PUSH_NOW(dst_ev, i_, done_created, 0); }
                if (active < c_limit) { uint64_t i_ = ctr++; HS_PUSH_NOW(HS_EV_POLL, i_, 0, 0); }
                break;
            }
            case HS_EV_REQ_SINK:
            case HS_EV_REQ_COUNTER:
                HS_EMIT(kind, bi, M.dst_id);
                HS_SINK(e_created);
                break;
            default: break;
            }
            if (SIMPLE) sticky_slow = HS_STICKY_SLOW();
        }
    }
#undef HS_STICKY_SLOW

    if (!valid) return;
    if (P.resume && S->done) return;        /* finished in an earlier window: outputs already final */
    if (FLAGS & HS_LF_BUCKETS) hs_bucket_flush(BK, r, 0u, bacc);   /* the current time bucket, at the run's end or a pause */
    if (FLAGS & HS_LF_BUCKET_PCT) status |= hs_bucket_status(BK, r);
    if (FLAGS & HS_LF_REC) {                /* Sink samples still staged, entry by entry (before st_fl moves) */
        if (smp_full) {
            const uint32_t g = (smp_pos == 0u ? P.sample_cap : smp_pos) - HS_SMP_GROUP;
            for (uint32_t q = 0; q < HS_SMP_GROUP - 1; ++q) *(uint4 *)(smp + g + q) = sh_smp[q][tid];
            *(uint4 *)(smp + g + HS_SMP_GROUP - 1) = sh_rec[(st_fl + HS_STAGE - 1u) % HS_STAGE][tid];
        } else if (smp_sync) {
            for (uint32_t q = 0; q < smp_pos % HS_SMP_GROUP; ++q) *(uint4 *)(smp + smp_pos - smp_pos % HS_SMP_GROUP + q) = sh_smp[q][tid];
        }
    }
    if ((FLAGS & HS_LF_REC) && svc_chunks) {
        /* service draw j, as the refill round computes it */
        auto service_draw = [&](uint64_t j) -> double {
            int64_t d = hs_seconds_to_ns(mean);
            if (expo && !trace_svc) { double u0 = 0.0, u1 = 0.0; hs_uniform_pair(seed, rid, sid_svc, j >> 1, &u0, &u1);
                                      d = hs_exp_latency_ns_r((j & 1) ? u1 : u0, lambda, lambda_recip); }
            if (expo && trace_svc) d = hs_seconds_to_ns(hs_div_by(trace_svc[(size_t)r * P.n_trace_svc + j], lambda, lambda_recip));
            return hs_ns_to_seconds(d);
        };
        /* The refill round has written every chunk below w_end.  Draws consumed after it (w_end .. n_svc - 1, a chunk
         * not generated whole yet) are still in the draw buffer and are written from there. */
        const uint64_t w_end = s_gen & ~(uint64_t)(HS_SVC_CHUNK - 1);
        uint32_t pos = svc_pos;
        for (uint64_t j = (uint64_t)n_svc; j > w_end; --j) {
            pos = (pos == 0u ? P.service_cap : pos) - 1u;
            svc_out[pos] = sh_svc[(j - 1) % HS_DRAW_BUF][tid];
        }
        /* Undo the write-ahead: the slots of draws n_svc .. w_end - 1 were written before their service started.
         * Each gets back what it held before this launch: the draw one ring pass earlier, or 0 if there was none (a
         * run that is not resumed starts from zeroed rings). */
        pos = svc_pos;
        for (uint64_t j = (uint64_t)n_svc; j < w_end; ++j) {
            svc_out[pos] = j >= P.service_cap ? service_draw(j - P.service_cap) : 0.0;
            pos = (pos + 1 == P.service_cap) ? 0u : pos + 1;
        }
    }
    if ((FLAGS & HS_LF_REC) && staged) {    /* drain what is still staged, record by record */
        while (st_fl != st_wr) {
            __stcs((uint4 *)(rec + rec_pos), sh_rec[st_fl % HS_STAGE][tid]);
            st_fl++; rec_pos = (rec_pos + 1 == P.record_cap) ? 0u : rec_pos + 1;
        }
    }

    /* ---- persist / publish --------------------------------------------- */
    /* derived counters: a tick is processed per consumed arrival time except the pending one;
     * every started service completes exactly once; a completion that forwards downstream is
     * counted by the Sink/Counter once its (same-timestamp) event has been processed. */
    const int64_t gen_count = (int64_t)arr_draws - 1;
    const int64_t skipped = S->skipped;
    const int64_t completed = n_svc - active;
    const int64_t rejected = S->rejected;
    int64_t received = (M.dst_id >= 0) ? completed : 0;
    int64_t pending_enq = 0;
    for (int i = 0; i < now_n; ++i) { if (nowq[i].kind == dst_ev) received--; if (nowq[i].kind == HS_EV_REQ_ENQUEUE) pending_enq++; }
    /* every payload's ENQUEUE is either accepted, dropped, still pending at this timestamp, or the one
     * that found the device ring full (the replica stops right there) */
    const int64_t accepted = (gen_count - skipped) - pending_enq - dropped - ((status & HS_ST_QUEUE_OVERFLOW) ? 1 : 0);
    S->now = now; S->ctr = ctr; S->processed = processed; S->hash = hash;
    S->tT = tT; S->iT = iT; S->arr_draws = arr_draws; S->gen_count = gen_count; S->prov_count = gen_count - skipped;
    S->tC = tC; S->iC = iC; S->svc_s = svc_s; S->c_created = c_created;
    S->svc_draws = (uint64_t)n_svc; S->accepted = accepted; S->dropped = dropped; S->completed = completed;
    S->total_service = total_service;
    S->received = received; S->sum = sum; S->comp = comp; S->sumsq = sumsq; S->mn = mn; S->mx = mx;
    S->q_head = q_head; S->q_len = q_len; S->active = active; S->status = status;
    S->n_smp = received; S->n_svc = n_svc; S->now_n = now_n; S->has_c = active > 0;
    S->rec_pos = rec_pos; S->smp_pos = smp_pos; S->svc_pos = svc_pos;
    S->done = paused ? 0 : 1;
    for (int i = 0; i < HS_NOW_CAP; ++i) S->nowq[i] = nowq[i];

    if (O.summaries) {
        hs_replica_summary s;
        s.events_processed = processed; s.final_time_ns = now;
        s.order_hash = (FLAGS & HS_LF_HASH) ? hash : 0ULL;
        s.next_sort_index = ctr; s.n_sink_samples = (M.dst_kind == HS_ENT_SINK) ? received : 0; s.n_service_samples = n_svc;
        s.heap_left = (tT != INT64_MAX) + active + now_n; s.status = status;
        O.summaries[r] = s;
    }
    if (O.stats) {
        hs_entity_stats *st = O.stats + (size_t)r * M.n_entities;
        hs_entity_stats a; a.c0 = gen_count; a.c1 = gen_count - skipped; a.c2 = 0; a.c3 = 0; a.f0 = a.f1 = a.f2 = a.f3 = 0.0;
        st[M.src_id] = a;
        a.c0 = accepted; a.c1 = dropped; a.c2 = completed; a.c3 = rejected; a.f0 = total_service;
        st[M.srv_id] = a;
        if (M.dst_id >= 0) {
            a.c0 = received; a.c1 = a.c2 = a.c3 = 0;
            if (M.dst_kind == HS_ENT_SINK) { a.f0 = hs_neumaier_result(sum, comp); a.f1 = sumsq; a.f2 = mn; a.f3 = mx; }
            else { a.f0 = a.f1 = a.f2 = a.f3 = 0.0; }
            st[M.dst_id] = a;
        }
    }
#undef HS_EMIT
#undef HS_RECORD
#undef HS_REFILL_ROUND
#undef HS_NEXT_ARRIVAL
#undef HS_NEXT_TICK
#undef HS_SERVICE_START
#undef HS_SINK
#undef HS_SMP_STORE
#undef HS_SVC_STORE
#undef HS_SVC_FLUSH
#undef HS_Q_PUSH
#undef HS_Q_POP
#undef HS_PUSH_NOW
#undef HS_C_PUSH
#undef HS_C_POP
#undef HS_CLT
}

#endif /* HS_LANE_ENGINE_CUH */
