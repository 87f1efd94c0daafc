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
#include "../../include/hs_b200.h"

#define HS_NOW_CAP 8
#define HS_LANE_THREADS 64
#define HS_DRAW_BUF_SUMMARY 16  /* precomputed draws per stream per lane (even)            */
#define HS_DRAW_BUF_RECORD 8    /* ... when the recorder staging shares the shared memory  */
#define HS_STAGE 16             /* staged event records per lane (recorder kernels)        */
#define HS_FLUSH 8              /* records per flush: 8 x 16 B = one 128 B line            */
#define HS_LF_HASH 1      /* maintain the order hash                         */
#define HS_LF_REC 2       /* write event records / sink / service samples    */
#define HS_LF_PROFILE 4   /* non-constant rate profile (Simpson + Brent path) */
#define HS_LF_SIMPLE 8    /* compile-time model: Poisson source without stop_after, exponential FIFO server with an
                             unbounded queue, Sink downstream, Philox draws -- the BASELINE configs[0]/[1] shape */

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

struct hs_lane_run {
    uint64_t seed, seed_stride;
    uint32_t rid_base, rid_stride;
    int64_t end_ns, window_end_ns;
    uint32_t n_replicas, index_base, replicas_per_cell;
    uint32_t record_cap, sample_cap, service_cap, ring, resume;
    int64_t max_events;                     /* INT64_MAX = unlimited */
    const double *trace_arr, *trace_svc;    /* externally supplied draws (hs_set_trace) or NULL */
    uint64_t n_trace_arr, n_trace_svc;
};

struct hs_lane_out {
    hs_replica_summary *summaries;
    hs_entity_stats *stats;
    hs_event_record *records;
    hs_sink_sample *samples;
    double *service;
    uint32_t *hist;                   /* [replica][HS_HIST_BINS] or NULL */
};

/* 256-bit global store: one full 32-byte sector per lane, written as two back-to-back 128-bit stores
 * (STG.E.128, the widest global store of sm_90a) to the two halves of the sector.  The recorder streams
 * are write-once per ring pass, so they are written with the streaming policy (st.global.cs,
 * HS_ST256_POLICY 2).  1 selects L1 no-allocate + an L2 evict-first cache policy, 0 the default
 * write-back policy; kept as a compile-time switch for A/B measurements.  tools/bench_lane.py on one
 * H100 80GB HBM3 (400 W power limit), record mode, 65 536 replicas: 2 -> 37.1e9, 1 -> 35.3e9,
 * 0 -> 32.2e9 events/s (profiles/h100_lane_store_policy_ab.txt). */
#ifndef HS_ST256_POLICY
#define HS_ST256_POLICY 2
#endif
#ifndef HS_LANE_PREDICATED
#define HS_LANE_PREDICATED 1    /* SIMPLE chains: state updates as selects + predicated memory operations (0: two branches) */
#endif
__device__ __forceinline__ void hs_st128(void *p, const uint4 a)
{
#if HS_ST256_POLICY == 1
    asm volatile("{\n\t.reg .b64 pol;\n\t"
                 "createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
                 "st.global.L1::no_allocate.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, pol;\n\t}"
#elif HS_ST256_POLICY == 2
    asm volatile("st.global.cs.v4.b32 [%0], {%1,%2,%3,%4};"
#else
    asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};"
#endif
                 :: "l"(p), "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w) : "memory");
}
__device__ __forceinline__ void hs_st256(void *p, const uint4 a, const uint4 b)
{
    hs_st128(p, a);
    hs_st128((uint4 *)p + 1, b);
}

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

template <int FLAGS>
__global__ void __launch_bounds__(HS_LANE_THREADS, 7)
hs_lane_kernel(hs_lane_model M, hs_lane_run P, hs_lane_state *__restrict__ states,
               hs_ring_entry *__restrict__ rings, hs_cont *__restrict__ conts, hs_lane_out O)
{
    constexpr uint32_t HS_DRAW_BUF = (FLAGS & HS_LF_REC) ? HS_DRAW_BUF_RECORD : HS_DRAW_BUF_SUMMARY;
    constexpr uint32_t STAGE_ROWS = (FLAGS & HS_LF_REC) ? HS_STAGE : 1;
    __shared__ int64_t sh_t[HS_DRAW_BUF][HS_LANE_THREADS];       /* arrival times A_k (ns)          */
    __shared__ double sh_svc[HS_DRAW_BUF][HS_LANE_THREADS];      /* service: Duration.to_seconds()  */
    /* recorder staging, [slot][lane]: a lane only ever touches its own 16-byte column, so neither the
     * per-event writes nor the flush reads conflict, whatever slot each lane is at.  A lane that holds a
     * full 128-byte group (8 records) writes it itself as four 256-bit stores (whole 32-byte sectors,
     * the four sectors of one line back to back).  Sink samples (16 B) and service times (8 B) are paired /
     * quadrupled the same way into one 32-byte sector per store. */
    __shared__ __align__(16) uint4 sh_rec[STAGE_ROWS][HS_LANE_THREADS];
    __shared__ __align__(16) uint4 sh_smp[(FLAGS & HS_LF_REC) ? HS_LANE_THREADS : 1];        /* first Sink sample of a pair */
    __shared__ double sh_sv[(FLAGS & HS_LF_REC) ? 3 : 1][HS_LANE_THREADS];                   /* first three service times of a quad */
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
    /* sample streams: *_sync <=> every earlier entry of the 32-byte sector being filled is staged in shared memory */
    const bool smp_pairs = (FLAGS & HS_LF_REC) && (P.sample_cap % 2u) == 0;
    const bool svc_quads = (FLAGS & HS_LF_REC) && (P.service_cap % 4u) == 0;
    bool smp_sync = false, svc_sync = false;
    hs_now_ev nowq[HS_NOW_CAP];

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
     * is regenerated and its first half skipped). */
    uint64_t a_gen = arr_draws, s_gen = (uint64_t)n_svc;
    int64_t t_gen = P.resume ? tT : 0;

    /* next arrival time from t (arrival_time_provider.py:66-82); a result < t would be
     * popped and skipped as "time travel" by the loop (simulation.py:479-489), after which the
     * Source never ticks again: INT64_MAX marks that dead source. */
#define HS_NEXT_ARRIVAL(T, TARGET) hs_lane_next_arrival<(FLAGS & HS_LF_PROFILE) != 0>((T), (TARGET), rate, rate_recip, profp)

    /* one converged refill round: each lane that has room generates the next Philox
     * pair of each stream and stores the precomputed draws */
#define HS_REFILL_ROUND()                                                                    \
    do {                                                                                     \
        if (!finished && (uint32_t)(a_gen - arr_draws) + 2u <= HS_DRAW_BUF) {                \
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
                sh_t[a_gen % HS_DRAW_BUF][tid] = t_gen;                                      \
            }                                                                                \
            t_gen = HS_NEXT_ARRIVAL(t_gen, g1_); a_gen++;                                    \
            sh_t[a_gen % HS_DRAW_BUF][tid] = t_gen;                                          \
        }                                                                                    \
        if (!finished && (uint32_t)(s_gen - (uint64_t)n_svc) + 2u <= HS_DRAW_BUF) {          \
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
        }                                                                                    \
    } while (0)

    /* Sink sample / service time into their rings, one whole 32-byte sector per global store: the first
     * entries of a sector wait in the lane's shared-memory column, the last one completes the 256-bit
     * store.  A sector that was begun before this launch (resume at an odd position) or rings whose
     * capacity is not a multiple of the sector are written entry by entry. */
#define HS_SMP_STORE(W)                                                                      \
    do {                                                                                     \
        const uint32_t p_ = smp_pos;                                                         \
        if (!(p_ & 1u)) smp_sync = smp_pairs;                                                \
        if (smp_sync) { if (!(p_ & 1u)) sh_smp[tid] = (W); else hs_st256(smp + (p_ - 1u), sh_smp[tid], (W)); } \
        else *(uint4 *)(smp + p_) = (W);                                                     \
        smp_pos = (p_ + 1 == P.sample_cap) ? 0u : p_ + 1;                                    \
    } while (0)
#define HS_SVC_STORE(V)                                                                      \
    do {                                                                                     \
        const uint32_t p_ = svc_pos, q_ = p_ & 3u; const double v_ = (V);                    \
        if (q_ == 0u) svc_sync = svc_quads;                                                  \
        if (svc_sync) {                                                                      \
            if (q_ < 3u) sh_sv[q_][tid] = v_;                                                \
            else { const uint64_t a_ = (uint64_t)__double_as_longlong(sh_sv[0][tid]), b_ = (uint64_t)__double_as_longlong(sh_sv[1][tid]), \
                                  c_ = (uint64_t)__double_as_longlong(sh_sv[2][tid]), d_ = (uint64_t)__double_as_longlong(v_);            \
                   hs_st256(svc_out + (p_ - 3u), make_uint4((uint32_t)a_, (uint32_t)(a_ >> 32), (uint32_t)b_, (uint32_t)(b_ >> 32)),      \
                            make_uint4((uint32_t)c_, (uint32_t)(c_ >> 32), (uint32_t)d_, (uint32_t)(d_ >> 32))); }                        \
        } else svc_out[p_] = v_;                                                             \
        svc_pos = (p_ + 1 == P.service_cap) ? 0u : p_ + 1;                                   \
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
    do { arr_draws++; tT = sh_t[arr_draws % HS_DRAW_BUF][tid];                               \
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
        /* SIMPLE: the three shared-memory operands of the next chain are requested first, so their
         * latency is covered by the flush below: next arrival time, next service time, queue head */
        int64_t tT_next = 0; double sv_next = 0.0; hs_ring_entry h; h.created = 0; h.idx = 0;
        if (SIMPLE) {
            tT_next = sh_t[(arr_draws + 1) % HS_DRAW_BUF][tid];
            sv_next = sh_svc[(uint32_t)((uint64_t)n_svc % HS_DRAW_BUF)][tid];
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            h = *my_head;                                    /* next queued request (meaningful if q_len > 0) */
        }
        if (FLAGS & HS_LF_REC) {
            /* a lane holding a full 128-byte group writes it itself: 8 reads of its own staging column,
             * four 256-bit stores (st_fl is a multiple of 8, so the group is rows 0-7 or 8-15) */
            if (staged && (st_wr - st_fl) >= HS_FLUSH) {
                const uint4 *src = &sh_rec[st_fl & (HS_STAGE - 1)][tid];
                uint4 *dst = (uint4 *)(rec + rec_pos);
#pragma unroll
                for (int g = 0; g < HS_FLUSH; g += 2)
                    hs_st256(dst + g, src[(size_t)g * HS_LANE_THREADS], src[(size_t)(g + 1) * HS_LANE_THREADS]);
                st_fl += HS_FLUSH; rec_pos = (rec_pos + HS_FLUSH == P.record_cap) ? 0u : rec_pos + HS_FLUSH;
            }
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
                /* Two forms of the same updates, chosen per kernel by A/B measurement (tools/bench_lane.py, with
                 * HS_LANE_PREDICATED=0/1 builds): selects + predicated memory operations (no branch, no reconvergence
                 * point, no register shuffling where the chains meet again) won without the recorder and with the
                 * order hash; with the recorder alone the two-branch form won (the predicated Sink block keeps more
                 * values live across the staged stores). */
                constexpr bool PREDICATED = HS_LANE_PREDICATED != 0 && (!(FLAGS & HS_LF_REC) || (FLAGS & HS_LF_HASH));
                if (PREDICATED) {
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
                } else {
                if (isA) {
                    /* Source: payload index c0, next SourceEvent index c0 + 1 (source.py:166-170) */
                    arr_draws++; tT = tT_next; iT = c0 + 1;
                    if (!start) {                                   /* Queue._handle_enqueue: the request waits */
                        hs_ring_entry e_; e_.created = now; e_.idx = c0;
                        ring[(q_head + q_len) & ring_mask] = e_;
                        if (q_empty) *my_head = e_;
                        q_len++;
                    }
                } else {
                    /* Server resumes after its yield, the Sink takes the request (server.py:255-273, common.py:36-44) */
                    total_service = HS_ADD(total_service, svc_s);
                    HS_SINK(c_created);
                    active = 0;
                    if (start) {                                    /* Queue._handle_poll: pop the head, prefetch the next */
                        q_head++; q_len--;
                        if (q_len == 0) q_head = 0;                 /* an empty queue restarts at slot 0 (hot lines stay in L2) */
                        if (q_len > 0) {
                            const hs_ring_entry *n_ = ring + (q_head & ring_mask);
                            asm volatile("cp.async.ca.shared.global [%0], [%1], 16;\n\tcp.async.commit_group;"
                                         :: "r"(my_head_s), "l"(n_) : "memory");
                        }
                    }
                }
                if (start) {
                    /* Server.handle_queued_event up to its yield (server.py:217-253): the scheduled
                     * ProcessContinuation takes the last index of the chain */
                    const double sv_ = sv_next;
                    if ((FLAGS & HS_LF_REC) && svc_out) HS_SVC_STORE(sv_);
                    n_svc++;
                    tC = now + hs_seconds_to_ns(sv_); iC = ctr - 1; c_created = start_created; svc_s = sv_; active = 1;
                }
                }
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
    if ((FLAGS & HS_LF_REC) && staged) {    /* drain what is still staged, record by record */
        while (st_fl != st_wr) {
            __stcs((uint4 *)(rec + rec_pos), sh_rec[st_fl % HS_STAGE][tid]);
            st_fl++; rec_pos = (rec_pos + 1 == P.record_cap) ? 0u : rec_pos + 1;
        }
    }
    if (FLAGS & HS_LF_REC) {                /* entries of a sector that is not complete yet */
        if (smp_sync && (smp_pos & 1u)) *(uint4 *)(smp + (smp_pos - 1u)) = sh_smp[tid];
        if (svc_sync) for (uint32_t q = 0; q < (svc_pos & 3u); ++q) svc_out[svc_pos - (svc_pos & 3u) + q] = sh_sv[q][tid];
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
#undef HS_Q_PUSH
#undef HS_Q_POP
#undef HS_PUSH_NOW
#undef HS_C_PUSH
#undef HS_C_POP
#undef HS_CLT
}

#endif /* HS_LANE_ENGINE_CUH */
