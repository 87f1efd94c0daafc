/* hs_warp_engine.cuh -- "warp engine": one WARP per replica, any lowered model
 * (sources, servers with concurrency c, sinks, counters, load balancers).
 *
 * Layout of one replica (contiguous block in HBM, staged into the warp's slice
 * of shared memory with TMA bulk copies -- cp.async.bulk + mbarrier -- when a
 * paused window is resumed, and written back with cp.async.bulk when the window
 * ends):
 *     [ header 128 B | entity state n x 96 B | future tier, SoA, S slots x 44 B |
 *       free-slot stack S x 2 B | now tier, 24 entries x 48 B ]
 * The pending-event set is kept in two tiers that together order exactly like the
 * reference's heap (time, then sort index):
 *   future tier  events scheduled later than `now` (SourceEvents, ProcessContinuations):
 *                S = 32 k slots, lane l owns slots l, l+32, ...; its minimum is found by a
 *                lane-parallel key scan + 5-step __shfl_xor_sync min-reduction and cached;
 *                a push only compares the new key with the cached minimum.
 *   now tier     events created at the current timestamp (the same-time protocol chain:
 *                ENQUEUE, NOTIFY, POLL, DELIVER, WORKER, SINK, _lb_response): a small array
 *                lane 0 scans by sort index.
 * Lane 0 executes the reference's handlers (scalar control flow over one entity's state)
 * and runs through a whole same-timestamp chain without involving the other lanes; the
 * warp only cooperates to extract the future-tier minimum (twice per request for a
 * Source -> Server path).  Queue contents live in per-server rings in HBM.
 *
 * This is the pop-invoke-push loop of happysimulator/core/simulation.py:449-505;
 * handlers: see oracle/hs_oracle.c for the one-to-one citations (identical
 * structure), and include/hs_b200.h for the event kinds.
 */
#ifndef HS_WARP_ENGINE_CUH
#define HS_WARP_ENGINE_CUH

#include "hs_sampler.h"
#include "hs_profile.h"
#include "hs_sketch.h"
#include "hs_kernel_params.cuh"
#include "hs_buckets.cuh"

#define HS_WF_HASH 1
#define HS_WF_REC 2
#define HS_WF_PROFILE 4    /* some Source has a non-constant rate profile (Simpson + Brent calls) */
#define HS_WF_HEAPTOP 8    /* thread engine: the heap's top levels live in shared memory (launches with several replicas per warp) */
#define HS_WF_LINKED 16    /* thread engine: a partition of a linked ParallelSimulation (REMOTE rows -> outbox, inbox drained at
                              launch, finished replicas run on, tie detection); compiled out of every other launch */
#define HS_WF_FAULTS 32    /* the model has FAULT rows (node faults): their bootstrap, the crashed-entity drop, cancelled pops and
                              the tie test; compiled out of every other launch */
#define HS_WF_BUCKETS 64   /* time buckets of the Sink / Probe samples (hs_set_buckets, hs_buckets.cuh); compiled out of every
                              other launch.  The row of a SINK / PROBE entity is the low word of its device row's d1 */
#define HS_WF_BUCKET_PCT 128 /* with HS_WF_BUCKETS: the buckets' p50 / p99 (hs_set_bucket_percentiles) */

/* The flag words (F < 256) the general engines are built for: FAULTS and BUCKETS always with the profile path (half the
 * kernels to build), BUCKETS never with the recorder, BUCKET_PCT only with BUCKETS.  hs_warp_kernel has none of the
 * thread-engine flags (hs_engine.cu launches it through a table indexed by the flag word; the thread engine's
 * predicates are next to its kernels). */
constexpr bool hs_general_built(int F)
{
    return (!(F & HS_WF_FAULTS) || (F & HS_WF_PROFILE)) && (!(F & HS_WF_BUCKETS) || ((F & HS_WF_PROFILE) && !(F & HS_WF_REC))) &&
           (!(F & HS_WF_BUCKET_PCT) || (F & HS_WF_BUCKETS));
}
constexpr bool hs_warp_built(int F) { return hs_general_built(F) && !(F & (HS_WF_HEAPTOP | HS_WF_LINKED)); }

struct __align__(16) hs_warp_hdr {      /* 128 B */
    int64_t now; uint64_t ctr; int64_t processed; uint64_t hash;
    int64_t n_smp, n_svc;
    uint32_t rec_pos, smp_pos, svc_pos, status;
    int32_t fel_n, done; int32_t now_n; uint32_t free_top;
    uint64_t np_cursor, py_cursor;      /* shared cursors of the externally supplied streams */
    uint32_t pad[8];
};

struct __align__(16) hs_went {          /* 96 B per entity */
    double d0;          /* effective rate / mean (cell override applied)          */
    double lambda;      /* SERVER: 1 / mean (exponential.py:36)                   */
    int32_t i0;         /* effective concurrency / arrival kind / strategy        */
    int32_t crashed;    /* Entity._crashed (faults/node_faults.py), set and cleared by FAULT events */
    int64_t pad1;
    union {
        struct { int64_t cur_ns; uint64_t arr_draws, key_draws; int64_t generated, provider; } src;
        struct { uint32_t q_head, q_len; int32_t active, pad; uint64_t svc_draws;
                 int64_t accepted, dropped, completed, rejected; double total_service; } srv;
        struct { int64_t received; double sum, comp, sumsq, mn, mx; } snk;
        struct { uint64_t rr_index; int64_t received, forwarded, in_flight, responses; } lb;
        struct { int64_t processed, added; } sk;
        struct { int64_t fired, cancelled; } flt;   /* FAULT: events fired / popped while cancelled */
        uint64_t raw[8];
    } u;
};

struct hs_wring_entry { int64_t created; uint64_t idx; int64_t key; };   /* 24 B */

/* PriorityQueue (components/queue_policy.py:189-287) of an HS_Q_PRIORITY server: a binary min-heap in slots
 * 0 .. q_len - 1 of the server's queue ring (q_head stays 0), ordered by (tab[routing key], insertion sequence) --
 * the reference's (priority, insert_order), a total order, so any heap pops what its heapq pops.  The sequence is the
 * server's accepted count at push time (PriorityQueue._insert_counter counts successful pushes), kept as 32 bits in
 * the upper half of the entry's key; compared modulo 2^32, it orders the entries exactly as long as the oldest and
 * the newest waiting request are fewer than 2^31 accepted requests apart.  The entry's idx (the payload's sort
 * index) is not the insertion order: a request delivered over a link carries the sending partition's index. */
__device__ __forceinline__ bool hs_pq_less(const double pa, const uint32_t sa, const double pb, const uint32_t sb)
{
    return pa < pb || (pa == pb && (int32_t)(sa - sb) < 0);
}
__device__ __forceinline__ double hs_pq_prio(const hs_wring_entry &e, const double *tab) { return tab[(int32_t)e.key]; }
__device__ __forceinline__ uint32_t hs_pq_seq(const hs_wring_entry &e) { return (uint32_t)((uint64_t)e.key >> 32); }

/* heappush of q (its key is the routing key, >= 0) as the seq-th accepted request into the heap of n entries */
__device__ __forceinline__ void hs_pq_push(hs_wring_entry *rg, uint32_t n, hs_wring_entry q, const uint32_t seq, const double *tab)
{
    q.key = (int64_t)(((uint64_t)seq << 32) | (uint64_t)(uint32_t)q.key);
    const double p = hs_pq_prio(q, tab);
    while (n > 0) {
        const uint32_t up = (n - 1) >> 1;
        const hs_wring_entry e = rg[up];
        if (!hs_pq_less(p, seq, hs_pq_prio(e, tab), hs_pq_seq(e))) break;
        rg[n] = e; n = up;
    }
    rg[n] = q;
}

/* heappop from the heap of n >= 1 entries: returns the root, its key the routing key again */
__device__ __forceinline__ hs_wring_entry hs_pq_pop(hs_wring_entry *rg, const uint32_t n, const double *tab)
{
    hs_wring_entry top = rg[0];
    top.key = (int32_t)top.key;
    const uint32_t m = n - 1;
    if (m > 0) {
        const hs_wring_entry last = rg[m];
        const double lp = hs_pq_prio(last, tab); const uint32_t ls = hs_pq_seq(last);
        uint32_t pos = 0;
        for (;;) {
            uint32_t c = 2 * pos + 1;
            if (c >= m) break;
            hs_wring_entry ce = rg[c]; double cp = hs_pq_prio(ce, tab); uint32_t cs = hs_pq_seq(ce);
            if (c + 1 < m) {
                const hs_wring_entry re = rg[c + 1]; const double rp = hs_pq_prio(re, tab); const uint32_t rs = hs_pq_seq(re);
                if (hs_pq_less(rp, rs, cp, cs)) { c = c + 1; ce = re; cp = rp; cs = rs; }
            }
            if (!hs_pq_less(cp, cs, lp, ls)) break;
            rg[pos] = ce; pos = c;
        }
        rg[pos] = last;
    }
    return top;
}

#define HS_W_NCAP 24
struct __align__(16) hs_wnow {          /* now-tier entry, 48 B */
    int64_t time; uint64_t idx; int64_t created; uint64_t aux;
    uint32_t m0; int32_t key; uint32_t hook; uint32_t pad;
};

struct hs_warp_model {
    const hs_entity_desc *ents;     /* device */
    const int32_t *backends, *key_table, *srv_index;
    const double *cell_d0; const int32_t *cell_i0;
    const hs_profile_desc *profiles;
    const int32_t *sketch_tables;   /* per-key hash results of the SKETCH rows                */
    const double *key_cdf;          /* cumulative key probabilities of the Zipf sources       */
    const double *profile_table;    /* STEP profile tables and the PriorityQueue servers' priority tables */
    uint64_t sk_total;              /* bytes of one replica's sketch states                   */
    uint32_t n_entities, n_cells, n_servers, fel_slots;   /* fel_slots = S, multiple of 32 */
    uint32_t block_bytes;           /* bytes of one replica block (multiple of 16)          */
    uint32_t n_backends, model_bytes; /* shared-memory copy of the model tables (per CTA)     */
    uint32_t outbox_cap, inbox_cap;   /* linked partitions (HS_ENT_REMOTE rows / link destination), else 0 */
    uint32_t fixed_slots, n_faults;   /* n_faults: FAULT rows, the last n_faults entities of the model.  fixed_slots: thread engine: every entity has at most ONE pending future event (sources: the next
                                         tick; servers with concurrency 1: the continuation), so its payload slot is its
                                         entity id -- no free-slot stack traffic on the heap's push / pop path */
};

/* ---- entity rows, shared by the warp and the thread engine ---------------- */

/* a row at the start of a run (the rest of it is zero): the cell's overrides, the CachingServer's unlimited
 * concurrency, the exponential rate and the Sink / Probe min / max sentinels */
__device__ __forceinline__ void hs_went_init(hs_went *e, const hs_entity_desc d, const hs_warp_model &M, uint32_t cell, uint32_t i)
{
    e->d0 = M.n_cells ? M.cell_d0[(size_t)cell * M.n_entities + i] : d.d0;
    e->i0 = M.n_cells ? M.cell_i0[(size_t)cell * M.n_entities + i] : d.i0;
    if (d.kind == HS_ENT_CACHE_SERVER) e->i0 = 0x7fffffff;          /* Entity.has_capacity() is True: no limit */
    e->lambda = (d.kind == HS_ENT_SERVER && d.i2 == HS_SVC_EXPONENTIAL) ? HS_DIV(1.0, e->d0) : 0.0;
    if (d.kind == HS_ENT_SINK || d.kind == HS_ENT_PROBE) {
        e->u.snk.mn = __longlong_as_double(0x7ff0000000000000LL);
        e->u.snk.mx = __longlong_as_double(0xfff0000000000000LL);
    }
}

/* what a row publishes */
__device__ __forceinline__ hs_entity_stats hs_went_stats(const hs_went *e, int32_t kind)
{
    hs_entity_stats a; a.c0 = a.c1 = a.c2 = a.c3 = 0; a.f0 = a.f1 = a.f2 = a.f3 = 0.0;
    switch (kind) {
    case HS_ENT_SOURCE: a.c0 = e->u.src.generated; a.c1 = e->u.src.provider; break;
    case HS_ENT_SERVER: a.c0 = e->u.srv.accepted; a.c1 = e->u.srv.dropped; a.c2 = e->u.srv.completed;
        a.c3 = e->u.srv.rejected; a.f0 = e->u.srv.total_service; break;
    case HS_ENT_CACHE_SERVER: a.c0 = e->u.srv.accepted; a.c1 = e->u.srv.dropped; a.c2 = e->u.srv.completed;
        a.c3 = e->u.srv.rejected; a.f0 = (double)e->u.srv.svc_draws; a.f1 = (double)e->u.srv.pad; break;   /* misses, hits, size */
    case HS_ENT_SINK: a.c0 = e->u.snk.received; a.f0 = hs_neumaier_result(e->u.snk.sum, e->u.snk.comp);
        a.f1 = e->u.snk.sumsq; a.f2 = e->u.snk.mn; a.f3 = e->u.snk.mx; break;
    case HS_ENT_COUNTER: case HS_ENT_REMOTE: a.c0 = e->u.snk.received; break;
    case HS_ENT_PROBE: a.c0 = e->u.snk.received; a.f0 = hs_neumaier_result(e->u.snk.sum, e->u.snk.comp);
        a.f2 = e->u.snk.mn; a.f3 = e->u.snk.mx; break;
    case HS_ENT_LB: a.c0 = e->u.lb.received; a.c1 = e->u.lb.forwarded; a.c2 = e->u.lb.in_flight;
        a.c3 = e->u.lb.responses; break;
    case HS_ENT_SKETCH: a.c0 = e->u.sk.processed; a.c1 = e->u.sk.added; break;
    }
    return a;
}
/* hs_went_stats of an instantiation that may hold FAULT rows (c0 fired, c1 popped while cancelled) */
template <int FLAGS>
__device__ __forceinline__ hs_entity_stats hs_went_stats_f(const hs_went *e, int32_t kind)
{
    if ((FLAGS & HS_WF_FAULTS) && kind == HS_ENT_FAULT) {
        hs_entity_stats a; a.c0 = e->u.flt.fired; a.c1 = e->u.flt.cancelled; a.c2 = a.c3 = 0; a.f0 = a.f1 = a.f2 = a.f3 = 0.0;
        return a;
    }
    return hs_went_stats(e, kind);
}

/* An event created during the run with the key (t, idx) of a FAULT event that is still pending (neither fired nor popped
 * cancelled): heapq would order the pair by its array layout (HS_ST_FAULT_TIE).  The FAULT rows are the model's last
 * n_faults rows, their keys are (l0, i3); row i's hs_went is at base + i * stride bytes. */
__device__ __forceinline__ bool hs_fault_tie(const hs_entity_desc *ENTS, uint32_t ne, uint32_t nf, int64_t t, uint64_t idx,
                                             const unsigned char *base, uint32_t stride)
{
    for (uint32_t i = ne - nf; i < ne; ++i)
        if (ENTS[i].l0 == t && (uint64_t)(uint32_t)ENTS[i].i3 == idx) {
            const hs_went *f = (const hs_went *)(base + (size_t)i * stride);
            if (f->u.flt.fired == 0 && f->u.flt.cancelled == 0) return true;
        }
    return false;
}

/* ---- PTX helpers: mbarrier + TMA 1-D bulk copies ------------------------- */
__device__ __forceinline__ uint32_t hs_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void hs_mbar_init(uint64_t *bar, uint32_t count)
{ asm volatile("mbarrier.init.shared.b64 [%0], %1;" ::"r"(hs_smem_u32(bar)), "r"(count) : "memory"); }

__device__ __forceinline__ void hs_mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    uint64_t state;
    asm volatile("mbarrier.arrive.expect_tx.release.cta.shared::cta.b64 %0, [%1], %2;"
                 : "=l"(state) : "r"(hs_smem_u32(bar)), "r"(bytes) : "memory");
    (void)state;
}

__device__ __forceinline__ void hs_mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        ::"r"(hs_smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ void hs_tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(hs_smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(hs_smem_u32(bar)) : "memory");
}

/* every thread that wrote the staged block through the generic proxy fences it
 * towards the async proxy before the (single-thread) bulk store is issued */
__device__ __forceinline__ void hs_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void hs_tma_store_1d(void *gmem_dst, const void *smem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gmem_dst), "r"(hs_smem_u32(smem_src)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

/* ---- the kernel --------------------------------------------------------- */

#define HS_W_EMPTY 0x7fffffffffffffffLL
#define HS_W_NONE 0xffffffffu

template <int FLAGS>
__global__ void __launch_bounds__(256)
hs_warp_kernel(hs_warp_model M, hs_kernel_run P, unsigned char *__restrict__ blocks,
               hs_wring_entry *__restrict__ rings, hs_kernel_out O, unsigned int *__restrict__ next_replica,
               typename hs_bucket_args_of<(FLAGS & HS_WF_BUCKETS) != 0, (FLAGS & HS_WF_BUCKET_PCT) != 0>::type BK)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t S = M.fel_slots;
    const uint32_t ne = M.n_entities;
    const uint32_t per_warp = 16u + M.block_bytes;          /* mbarrier slot + block */
    /* The model tables are read on every event by lane 0 in a dependent chain: keep one copy per CTA in
     * shared memory (entity rows, server ring index, load-balancer backend lists) instead of going to L2. */
    const hs_entity_desc *ENTS = M.ents;                    /* models too large for the copy stay in HBM/L2 */
    const int32_t *SRVIDX = M.srv_index, *BACKENDS = M.backends;
    if (M.model_bytes) {
        hs_entity_desc *es = (hs_entity_desc *)smem_raw;
        int32_t *si = (int32_t *)(smem_raw + (size_t)ne * sizeof(hs_entity_desc));
        int32_t *bs = si + ne;
        for (uint32_t i = threadIdx.x; i < ne * (uint32_t)(sizeof(hs_entity_desc) / 4); i += blockDim.x)
            ((uint32_t *)es)[i] = ((const uint32_t *)M.ents)[i];
        for (uint32_t i = threadIdx.x; i < ne; i += blockDim.x) si[i] = M.srv_index[i];
        for (uint32_t i = threadIdx.x; i < M.n_backends; i += blockDim.x) bs[i] = M.backends[i];
        __syncthreads();
        ENTS = es; SRVIDX = si; BACKENDS = bs;
    }
    unsigned char *base = smem_raw + M.model_bytes + (size_t)warp * per_warp;
    uint64_t *mbar = (uint64_t *)base;
    unsigned char *blk = base + 16;
    hs_warp_hdr *H = (hs_warp_hdr *)blk;
    hs_went *E = (hs_went *)(blk + sizeof(hs_warp_hdr));
    unsigned char *felp = blk + sizeof(hs_warp_hdr) + (size_t)ne * sizeof(hs_went);
    int64_t *f_time = (int64_t *)felp;
    uint64_t *f_idx = (uint64_t *)(felp + (size_t)S * 8);
    int64_t *f_created = (int64_t *)(felp + (size_t)S * 16);
    uint64_t *f_aux = (uint64_t *)(felp + (size_t)S * 24);
    uint32_t *f_m0 = (uint32_t *)(felp + (size_t)S * 32);   /* kind | ent << 8              */
    int32_t *f_key = (int32_t *)(felp + (size_t)S * 36);
    uint32_t *f_hook = (uint32_t *)(felp + (size_t)S * 40); /* (lb_hook + 1) | poll << 31   */
    uint16_t *f_free = (uint16_t *)(felp + (size_t)S * 44); /* stack of free future slots   */
    hs_wnow *N = (hs_wnow *)(felp + (((size_t)S * 46 + 15) / 16) * 16);

    if (lane == 0) hs_mbar_init(mbar, 1);
    __syncwarp();
    uint32_t phase = 0;
    const bool windowed = (P.window_end_ns >= 0 && P.window_end_ns < P.end_ns);

    while (true) {
        uint32_t r = 0;
        if (lane == 0) r = atomicAdd(next_replica, 1u);
        r = __shfl_sync(0xffffffffu, r, 0);
        if (r >= P.n_replicas) break;

        const uint32_t gidx = P.index_base + r;
        const uint64_t seed = P.seed + (uint64_t)gidx * P.seed_stride;
        const uint32_t rid = P.rid_base + gidx * P.rid_stride;
        unsigned char *gblk = blocks + (size_t)r * M.block_bytes;
        hs_wring_entry *ring0 = rings + (size_t)r * M.n_servers * P.ring;
        const uint32_t ring_mask = P.ring - 1u;

        /* ---- stage the replica into shared memory -------------------------- */
        if (P.resume) {
            if (lane == 0) {
                hs_mbar_expect_tx(mbar, M.block_bytes);
                hs_tma_load_1d(blk, gblk, M.block_bytes, mbar);
            }
            hs_mbar_wait(mbar, phase);
            phase ^= 1u;
            __syncwarp();
            if (H->done) continue;                      /* finished in an earlier window */
        } else {
            for (uint32_t i = lane; i < M.block_bytes / 8; i += 32) ((uint64_t *)blk)[i] = 0ull;
            __syncwarp();
            for (uint32_t i = lane; i < S; i += 32) { f_time[i] = HS_W_EMPTY; f_free[i] = (uint16_t)(S - 1 - i); }
            const uint32_t cell = M.n_cells ? (gidx / P.replicas_per_cell) % M.n_cells : 0u;
            for (uint32_t i = lane; i < ne; i += 32) hs_went_init(&E[i], ENTS[i], M, cell, i);
            __syncwarp();
            if (lane == 0) {
                H->hash = HS_HASH_INIT;
                H->free_top = S;
                /* Simulation.__init__: source.start() in order; bootstrap indices come from the
                 * global counter (simulation.py:77,145-154), run() restarts the per-heap one at 0. */
                uint64_t boot = 0; int nf = 0;
                for (uint32_t i = 0; i < ne; ++i) {
                    if (ENTS[i].kind != HS_ENT_SOURCE) continue;
                    hs_went *e = &E[i];
                    double target = 1.0;
                    if (e->i0 == HS_ARR_POISSON && P.trace_arr) {
                        if (H->np_cursor >= P.n_trace_arr) { H->status |= HS_ST_TRACE_EXHAUSTED; break; }
                        target = P.trace_arr[(size_t)r * P.n_trace_arr + H->np_cursor++]; e->u.src.arr_draws++;
                    } else if (e->i0 == HS_ARR_POISSON) {
                        double u = hs_uniform(seed, rid, HS_STREAM_ARRIVAL | (i << 8), e->u.src.arr_draws++);
                        target = hs_exp1(u);
                    }
                    const int32_t pi = ENTS[i].i3;
                    int64_t first;
                    if ((FLAGS & HS_WF_PROFILE) && pi > 0) first = hs_next_arrival_profile_ns(&M.profiles[pi - 1], 0, target);
                    else first = hs_next_arrival_ns(0, target, e->d0);
                    if (first == HS_T_EXHAUSTED) continue;      /* source.start(): RuntimeError, no tick */
                    e->u.src.cur_ns = first;
                    if (H->free_top == 0) { H->status |= HS_ST_FEL_OVERFLOW; break; }
                    const uint32_t sl = f_free[--H->free_top];
                    f_time[sl] = e->u.src.cur_ns; f_idx[sl] = boot++; f_m0[sl] = HS_EV_SOURCE_TICK | (i << 8);
                    f_key[sl] = -1; f_hook[sl] = 0; nf++;
                }
                /* FaultSchedule.start() after the sources and probes (simulation.py:162-169): one Event.once per fault
                 * event, its sort index taken from the same global counter (carried in the row) */
                if (FLAGS & HS_WF_FAULTS)
                    for (uint32_t i = ne - M.n_faults; i < ne; ++i) {
                        if (H->free_top == 0) { H->status |= HS_ST_FEL_OVERFLOW; break; }
                        const uint32_t sl = f_free[--H->free_top];
                        f_time[sl] = ENTS[i].l0; f_idx[sl] = (uint64_t)(uint32_t)ENTS[i].i3; f_m0[sl] = HS_EV_FAULT | (i << 8);
                        f_key[sl] = -1; f_hook[sl] = 0; f_created[sl] = 0; f_aux[sl] = 0ull; nf++;
                    }
                H->fel_n = nf; H->ctr = 0;
            }
            __syncwarp();
        }

        hs_event_record *rec = (FLAGS & HS_WF_REC) && O.records ? O.records + (size_t)r * P.record_cap : nullptr;
        hs_sink_sample *smp = (FLAGS & HS_WF_REC) && O.samples ? O.samples + (size_t)r * P.sample_cap : nullptr;
        double *svc_out = (FLAGS & HS_WF_REC) && O.service ? O.service + (size_t)r * P.service_cap : nullptr;
        auto *const bacc = hs_bucket_accs(BK, blk);     /* HS_WF_BUCKETS: the rows' current time buckets, in the staged block */
        if (lane == 0) hs_bucket_begin(BK, bacc);

        /* ---- pop-invoke-push --------------------------------------------------- */
        bool paused = false;
        /* cached minimum of the future tier (valid on lane 0) */
        int64_t ft = HS_W_EMPTY; uint64_t fi = ~0ull; uint32_t fs = HS_W_NONE;
        bool rescan = true;
        while (true) {
            if (rescan) {
                /* lane-parallel scan + shuffle min-reduction over (time, sort_index) */
                int64_t bt = HS_W_EMPTY; uint64_t bi = ~0ull; uint32_t bs = HS_W_NONE;
                for (uint32_t s2 = lane; s2 < S; s2 += 32) {
                    const int64_t t = f_time[s2];
                    if (t != HS_W_EMPTY) {
                        const uint64_t ix = f_idx[s2];
                        if (t < bt || (t == bt && ix < bi)) { bt = t; bi = ix; bs = s2; }
                    }
                }
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) {
                    const int64_t ot = __shfl_xor_sync(0xffffffffu, bt, d);
                    const uint64_t oi = __shfl_xor_sync(0xffffffffu, bi, d);
                    const uint32_t os = __shfl_xor_sync(0xffffffffu, bs, d);
                    if (ot < bt || (ot == bt && (oi < bi || (oi == bi && os < bs)))) { bt = ot; bi = oi; bs = os; }
                }
                ft = bt; fi = bi; fs = bs;
                rescan = false;
            }
            int go = 0;        /* 0 stop, 1 extract the future-tier minimum, 2 paused */
            if (lane == 0) {
                uint64_t ctr = H->ctr;
                int now_n = H->now_n;
                /* ---- lane 0 runs the same-timestamp chain on its own -------------- */
                while (true) {
                    const int64_t now0 = H->now;
                    if (!(now0 <= P.end_ns) || (H->status & (HS_ST_QUEUE_OVERFLOW | HS_ST_FEL_OVERFLOW | HS_ST_TRACE_EXHAUSTED))) { go = 0; break; }
                    if (H->processed >= P.max_events) { H->status |= HS_ST_EVENT_LIMIT; go = 0; break; }
                    /* next event: minimum of the now tier, unless the future minimum sorts first */
                    int nb = -1; int64_t nt = HS_W_EMPTY; uint64_t ni = ~0ull;
                    for (int k = 0; k < now_n; ++k) {
                        const int64_t t = N[k].time; const uint64_t ix = N[k].idx;
                        if (t < nt || (t == nt && ix < ni)) { nt = t; ni = ix; nb = k; }
                    }
                    if (nb < 0 || (fs != HS_W_NONE && (ft < nt || (ft == nt && fi < ni)))) {
                        if (fs == HS_W_NONE) { go = 0; break; }                 /* heap exhausted */
                        if (windowed && ft > P.window_end_ns) { go = 2; break; }
                        go = 1; break;
                    }
                    if (windowed && nt > P.window_end_ns) { go = 2; break; }
                    /* ---- pop from the now tier ---- */
                    const hs_wnow ev = N[nb];
                    now_n--; N[nb] = N[now_n];
                    H->fel_n--;
                    if ((FLAGS & HS_WF_FAULTS) && (ev.m0 & 0xffu) == HS_EV_FAULT && ENTS[ev.m0 >> 8].i2) {
                        E[ev.m0 >> 8].u.flt.cancelled++;  /* a cancelled event: counted, not processed (simulation.py:475-477) */
                        continue;
                    }
                    if (ev.time < now0) continue;     /* "time travel": skipped (simulation.py:479-489) */
                    const int64_t now = ev.time;
                    const uint64_t bi = ev.idx;
                    const int kind = (int)(ev.m0 & 0xffu);
                    const uint32_t ent = ev.m0 >> 8;
                    const int64_t e_created = ev.created;
                    const uint64_t e_aux = ev.aux;
                    const int32_t e_key = ev.key;
                    const uint32_t e_hook = ev.hook;
                    H->now = now;
                    if (FLAGS & HS_WF_HASH) H->hash = hs_hash_step(H->hash, now, hs_record_word1(bi, (uint32_t)kind, ent));
                    if ((FLAGS & HS_WF_REC) && rec) {
                        hs_event_record rc; rc.time_ns = now; rc.sort_index = (uint32_t)bi; rc.kind = (uint8_t)kind;
                        rc.pad = 0; rc.entity = (uint16_t)ent;
                        rec[H->rec_pos] = rc; H->rec_pos = (H->rec_pos + 1 == P.record_cap) ? 0u : H->rec_pos + 1;
                    }
                    H->processed++;
                    hs_went *X = &E[ent];

                    /* push: an event at (or before) `now` joins the now tier, a later one the future
                     * tier (free slot from the stack; the cached minimum is updated in place) */
#define HS_W_PUSH(TIME, IDX, KIND, ENT, CREATED, AUX, KEY, HOOK)                                         \
    do {                                                                                                 \
        const int64_t t_ = (TIME);                                                                       \
        if ((FLAGS & HS_WF_FAULTS) && hs_fault_tie(ENTS, ne, M.n_faults, t_, (uint64_t)(IDX),            \
                                                   (const unsigned char *)E, (uint32_t)sizeof(hs_went))) \
            H->status |= HS_ST_FAULT_TIE;                                                                \
        if (t_ <= now) {                                                                                 \
            if (now_n >= HS_W_NCAP) H->status |= HS_ST_FEL_OVERFLOW;                                     \
            else { hs_wnow n_; n_.time = t_; n_.idx = (IDX); n_.created = (CREATED); n_.aux = (AUX);     \
                   n_.m0 = (uint32_t)(KIND) | ((uint32_t)(ENT) << 8); n_.key = (KEY); n_.hook = (HOOK); n_.pad = 0; \
                   N[now_n++] = n_; H->fel_n++; }                                                        \
        } else if (H->free_top == 0) H->status |= HS_ST_FEL_OVERFLOW;                                    \
        else {                                                                                           \
            const uint32_t s_ = f_free[--H->free_top]; const uint64_t i2_ = (IDX);                       \
            f_idx[s_] = i2_; f_created[s_] = (CREATED); f_aux[s_] = (AUX);                               \
            f_m0[s_] = (uint32_t)(KIND) | ((uint32_t)(ENT) << 8); f_key[s_] = (KEY); f_hook[s_] = (HOOK); \
            f_time[s_] = t_; H->fel_n++;                                                                 \
            if (fs == HS_W_NONE || t_ < ft || (t_ == ft && (i2_ < fi || (i2_ == fi && s_ < fs)))) { ft = t_; fi = i2_; fs = s_; } \
        }                                                                                                \
    } while (0)
#define HS_W_D (ENTS[ent])
#define HS_W_ENT(I) (&E[(I)])
#include "hs_handlers.inc"
#undef HS_W_ENT
#undef HS_W_D
#undef HS_W_PUSH
                }
                /* ---- extract the future-tier minimum into the now tier ------------- */
                if (go == 1) {
                    if (now_n >= HS_W_NCAP) { H->status |= HS_ST_FEL_OVERFLOW; go = 0; }
                    else {
                        hs_wnow n_; n_.time = ft; n_.idx = fi; n_.created = f_created[fs]; n_.aux = f_aux[fs];
                        n_.m0 = f_m0[fs]; n_.key = f_key[fs]; n_.hook = f_hook[fs]; n_.pad = 0;
                        N[now_n++] = n_;
                        f_time[fs] = HS_W_EMPTY;
                        f_free[H->free_top++] = (uint16_t)fs;
                    }
                }
                H->ctr = ctr; H->now_n = now_n;
            }
            go = __shfl_sync(0xffffffffu, go, 0);
            __syncwarp();
            if (go == 2) paused = true;
            if (go != 1) break;
            rescan = true;
        }

        /* ---- publish + write the block back -------------------------------- */
        if (lane == 0) {
            hs_bucket_end(BK, r, bacc);                 /* every row's current time bucket, at the run's end or a pause */
            if (FLAGS & HS_WF_BUCKET_PCT) H->status |= hs_bucket_status(BK, r);
            H->done = paused ? 0 : 1;
            if (O.summaries) {
                hs_replica_summary s;
                s.events_processed = H->processed; s.final_time_ns = H->now;
                s.order_hash = (FLAGS & HS_WF_HASH) ? H->hash : 0ull;
                s.next_sort_index = H->ctr; s.n_sink_samples = H->n_smp; s.n_service_samples = H->n_svc;
                s.heap_left = H->fel_n; s.status = H->status;
                O.summaries[r] = s;
            }
        }
        __syncwarp();
        if (O.stats)
            for (uint32_t i = lane; i < ne; i += 32) O.stats[(size_t)r * ne + i] = hs_went_stats_f<FLAGS>(&E[i], ENTS[i].kind);
        hs_fence_async_smem();
        __syncwarp();
        if (lane == 0) hs_tma_store_1d(gblk, blk, M.block_bytes);
        __syncwarp();
    }
}

#endif /* HS_WARP_ENGINE_CUH */
