/* hs_thread_engine.cuh -- "thread engine": one THREAD per replica for ANY lowered model
 * (load-balanced farms, tandem queues, several sources, probes ...).
 *
 * The warp engine gives a replica a whole warp but its handlers are scalar control flow, so 31
 * lanes idle; here every lane runs its own replica.  A replica's state cannot live in registers
 * (a 64-server farm is ~10 KB), so it stays in a contiguous per-replica block in HBM
 *     [ header 128 B | entities n x 128 B (state 96 B + own payload 32 B) | heap keys S x 16 B | payloads S x 32 B |
 *       free-slot stack S x 2 B | now-tier overflow 24 x 48 B ]
 * that only this thread touches (nothing to stage or synchronise; a paused window resumes from the
 * same bytes).  Pending events are kept in two tiers that together order exactly like the
 * reference's heap (time, then sort index):
 *   now tier     events created at the current timestamp (the same-time protocol chain ENQUEUE,
 *                NOTIFY, POLL, DELIVER, WORKER, SINK, _lb_response): the first HS_T_KS entries of
 *                every thread sit in shared memory ([entry][16-byte chunk][thread], conflict-free),
 *                deeper ones (rare: many events on one nanosecond) overflow to the block in HBM;
 *   future heap  SourceEvents / ProcessContinuations: a 4-ary min-heap of 16-byte keys
 *                (time, sort_index << 16 | payload slot) -- the four children of a node are one
 *                64-byte aligned line, so a pop costs log4(n) dependent line reads -- with the
 *                32-byte payloads parked in slots; the root key is cached in registers.
 * Threads of a warp run different handlers, so everything expensive is hoisted to where they are
 * converged again: the pop, the loads of the model row and the entity state (handlers work on a
 * private copy, written back after the switch), the random draw (phase B of hs_handlers.inc) and
 * the heap insertion of the (at most one) future event an event creates.
 *
 * Small ensembles do not fill the machine with 32 replicas per warp, and a warp's iteration takes as
 * long as the sum of the distinct paths its lanes take: the launch spreads the replicas over as many
 * warps as fit (P.lane_stride lanes per replica, the surplus lanes exit at once).
 *
 * Bound (ncu, profiles/r02c_ncu_thread_lb64.txt, the 64-server farm at 8 replicas per warp): exposed load latency and
 * dependent-instruction latency at 128 registers -- 2.4 long-scoreboard + 2.5 fixed-latency stall cycles per issued
 * instruction, 43 % issue active, 4.3 of the 8 lanes active on average, 50 warp-instructions per event (round 1: 136 at
 * 2.4 lanes) -- not bandwidth: DRAM runs at 0.43 TB/s.
 * Sort indices are packed above a 16-bit slot number in the heap keys: at most 2^48 events per replica and
 * 65 535 concurrently pending future events.
 */
#ifndef HS_THREAD_ENGINE_CUH
#define HS_THREAD_ENGINE_CUH

#include "hs_warp_engine.cuh"       /* hs_warp_hdr, hs_went and its init / publish, hs_wnow, hs_wring_entry, hs_warp_model */

#define HS_THREAD_BLOCK 64
#define HS_T_KS 4                   /* now-tier entries per replica held in shared memory */
#ifndef HS_T_ARITY
#define HS_T_ARITY 4                /* heap fan-out: the children of a node are one aligned line of ARITY keys */
#endif
#ifndef HS_T_MINBLOCKS
#define HS_T_MINBLOCKS 8             /* 8 x 64 threads x 128 registers = the register file */
#endif
#define HS_T_LEAD ((HS_T_ARITY - 1) * 16u)   /* bytes in front of heap key 0 */
#define HS_T_SHIFT (HS_T_ARITY == 8 ? 3 : 2)
#define HS_EV_REQ_ANY 0xffu         /* private: "request for entity `ent`", kind resolved when popped */

struct __align__(16) hs_tkey { int64_t time; uint64_t k2; };                 /* k2 = sort_index << 16 | slot */
struct __align__(16) hs_tpay { int64_t created; uint64_t aux; uint32_t m0; int32_t key; uint32_t hook, pad; };

/* One 128-byte line per entity: its state and, next to it, the payload of ITS pending future event (entity-owned slots,
 * hs_warp_model.fixed_slots: a source's next tick, a concurrency-1 server's continuation).  A pop then finds the payload
 * and the state of the entity it is for in the same line -- one miss instead of two or three (a 96-byte state at a
 * 96-byte stride straddles two lines half of the time) -- and these misses are what the kernel waits for. */
struct __align__(16) hs_tent { hs_went w; hs_tpay pay; };
static_assert(sizeof(hs_tent) == 128, "one line per entity");

struct hs_thread_layout { uint32_t keys, pay, free_, spill, total; };

__host__ __device__ inline hs_thread_layout hs_thread_offsets(uint32_t ne, uint32_t S)
{
    hs_thread_layout L;
    L.keys = (uint32_t)sizeof(hs_warp_hdr) + ne * (uint32_t)sizeof(hs_tent);      /* the header is one line too */
    L.pay = L.keys + (HS_T_LEAD + (S + HS_T_ARITY) * 16u + 127u) / 128u * 128u;   /* the children ARITY k + 1 .. ARITY k + ARITY share one aligned line */
    L.free_ = L.pay + S * 32u;
    L.spill = L.free_ + (S * 2u + 15u) / 16u * 16u;
    L.total = (L.spill + HS_W_NCAP * (uint32_t)sizeof(hs_wnow) + 127u) / 128u * 128u;
    return L;
}

#define HS_T_LT(T1, I1, T2, I2) ((T1) < (T2) || ((T1) == (T2) && (I1) < (I2)))

__device__ __forceinline__ void hs_prefetch(const void *p) { asm volatile("prefetch.global.L1 [%0];" :: "l"(p)); }


template <int FLAGS>
__device__ __forceinline__ void
hs_thread_body(const hs_warp_model &M, const hs_kernel_run &P, unsigned char *__restrict__ blocks,
               hs_wring_entry *__restrict__ rings, const hs_kernel_out &O,
               const typename hs_bucket_args_of<(FLAGS & HS_WF_BUCKETS) != 0, (FLAGS & HS_WF_BUCKET_PCT) != 0>::type BK)
{
    /* dynamic shared memory of a block: [ now tier: HS_T_KS x 3 chunks x rpb columns | heap top: P.heap_top keys x rpb columns ],
     * rpb = replicas (columns) of the block.  The now tier is sized by the columns in use (it was 64 wide whatever the
     * launch): shared memory is carved out of L1, and L1 is where the replicas' state lives -- configs[3] at one replica per
     * warp 1.30e9 -> 1.37e9 events/s, configs[2] at 8 per warp 9.0e9 -> 9.25e9 from this alone. */
    extern __shared__ uint4 hs_t_dyn[];
    const uint32_t rpb = HS_THREAD_BLOCK / P.lane_stride;            /* replica columns per block */
    uint4 *const Ns = hs_t_dyn;
    uint4 *const Ktop = hs_t_dyn + HS_T_KS * 3 * rpb;    /* the heap's top levels: [key index][replica column of the block] */
    const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gtid % P.lane_stride) return;                    /* surplus lanes (see above) */
    const int tid = (int)(threadIdx.x / P.lane_stride);  /* this replica's column of the shared now tier */
    const uint32_t r = gtid / P.lane_stride;
    if (r >= P.n_replicas) return;
    const uint32_t S = M.fel_slots;                      /* heap capacity */
    const uint32_t ne = M.n_entities;
    const hs_entity_desc *ENTS = M.ents;
    const int32_t *BACKENDS = M.backends;
    const hs_thread_layout L = hs_thread_offsets(ne, S);

    unsigned char *blk = blocks + (size_t)r * M.block_bytes;
    hs_warp_hdr *Hg = (hs_warp_hdr *)blk;
    hs_tent *E = (hs_tent *)(blk + sizeof(hs_warp_hdr));
    hs_tkey *K = (hs_tkey *)(blk + L.keys + HS_T_LEAD);
    hs_tpay *PAY = (hs_tpay *)(blk + L.pay);
    auto pay_at = [&](const uint32_t slot) -> hs_tpay * { return M.fixed_slots ? &E[slot].pay : &PAY[slot]; };
    uint16_t *FREE = (uint16_t *)(blk + L.free_);
    hs_wnow *Ng = (hs_wnow *)(blk + L.spill);
    auto *const bacc = hs_bucket_accs(BK, blk);          /* HS_WF_BUCKETS: the rows' current time buckets, after the block's own layout */

    /* Heap keys: the first P.heap_top (whole top levels) live in shared memory for the duration of the launch -- a pop's
     * sift-down walks the top of the heap every time, and in global memory every level is a dependent L2/DRAM round
     * trip; they are loaded on resume and written back at the end (the block in HBM stays the resumable image).
     * Compiled in (HS_WF_HEAPTOP) for launches with several replicas per warp: measured +5-7 % on the 64-server farm;
     * with one replica per warp the few resident heaps already sit in L1 and the extra addressing costs 10 %. */
    const uint32_t TOP = (FLAGS & HS_WF_HEAPTOP) ? P.heap_top : 0u;
    auto kload = [&](const uint32_t i) -> hs_tkey {
        if ((FLAGS & HS_WF_HEAPTOP) && i < TOP) { const uint4 q = Ktop[i * rpb + (uint32_t)tid]; hs_tkey k;
                       k.time = (int64_t)((uint64_t)q.x | ((uint64_t)q.y << 32)); k.k2 = (uint64_t)q.z | ((uint64_t)q.w << 32); return k; }
        return K[i];
    };
    auto kstore = [&](const uint32_t i, const hs_tkey &k) {
        if ((FLAGS & HS_WF_HEAPTOP) && i < TOP) Ktop[i * rpb + (uint32_t)tid] = make_uint4((uint32_t)(uint64_t)k.time, (uint32_t)((uint64_t)k.time >> 32), (uint32_t)k.k2, (uint32_t)(k.k2 >> 32));
        else K[i] = k;
    };

    const uint32_t gidx = P.index_base + r;
    const uint64_t seed = P.seed + (uint64_t)gidx * P.seed_stride;
    const uint32_t rid = P.rid_base + gidx * P.rid_stride;
    hs_wring_entry *ring0 = rings + (size_t)r * M.n_servers * P.ring;
    const uint32_t ring_mask = P.ring - 1u;
    const bool windowed = (P.window_end_ns >= 0 && P.window_end_ns < P.end_ns);

    /* entry k of the now tier: three 16-byte chunks, in shared memory (chunk stride = one row of the block)
     * for k < HS_T_KS, in the replica block (contiguous) beyond */
    union now_u { hs_wnow e; uint4 q[3]; };
    auto now_store = [&](int k, const hs_wnow &v) {
        now_u u; u.e = v;
        if (k < HS_T_KS) {
            Ns[(k * 3 + 0) * rpb + tid] = u.q[0];
            Ns[(k * 3 + 1) * rpb + tid] = u.q[1];
            Ns[(k * 3 + 2) * rpb + tid] = u.q[2];
        } else {
            uint4 *g = (uint4 *)&Ng[k]; g[0] = u.q[0]; g[1] = u.q[1]; g[2] = u.q[2];
        }
    };
    auto now_load = [&](int k) -> hs_wnow {
        now_u u;
        if (k < HS_T_KS) {
            u.q[0] = Ns[(k * 3 + 0) * rpb + tid];
            u.q[1] = Ns[(k * 3 + 1) * rpb + tid];
            u.q[2] = Ns[(k * 3 + 2) * rpb + tid];
        } else {
            const uint4 *g = (const uint4 *)&Ng[k]; u.q[0] = g[0]; u.q[1] = g[1]; u.q[2] = g[2];
        }
        return u.e;
    };
    auto now_key = [&](int k, int64_t &t, uint64_t &ix) {
        const uint4 a = (k < HS_T_KS) ? Ns[(k * 3) * rpb + tid] : *(const uint4 *)&Ng[k];
        t = (int64_t)((uint64_t)a.x | ((uint64_t)a.y << 32)); ix = (uint64_t)a.z | ((uint64_t)a.w << 32);
    };

    hs_warp_hdr hdr;                                     /* working copy of the header */
    hs_warp_hdr *H = &hdr;
    int64_t h_now = 0, h_processed = 0; uint64_t h_hash = 0; int32_t h_fel = 0;   /* its hot fields, in registers (see below) */
    if (P.resume) {
        hdr = *Hg;
        if (hdr.done && !((FLAGS & HS_WF_LINKED) && P.linked)) return;       /* a linked partition's next window: the end time has moved on, events may have arrived */
        h_now = H->now; h_processed = H->processed; h_hash = H->hash; h_fel = H->fel_n;
        for (uint32_t i = 0; i < TOP && i < hdr.free_top + HS_T_ARITY; ++i) {      /* the heap's top levels (free_top = heap size) */
            const hs_tkey k = K[i];
            Ktop[i * rpb + (uint32_t)tid] = make_uint4((uint32_t)(uint64_t)k.time, (uint32_t)((uint64_t)k.time >> 32), (uint32_t)k.k2, (uint32_t)(k.k2 >> 32));
        }
        for (int k = 0; k < hdr.now_n && k < HS_T_KS; ++k) {
            const uint4 *g = (const uint4 *)&Ng[k];
            Ns[(k * 3 + 0) * rpb + tid] = g[0];
            Ns[(k * 3 + 1) * rpb + tid] = g[1];
            Ns[(k * 3 + 2) * rpb + tid] = g[2];
        }
    } else {
        for (uint32_t i = 0; i < L.keys / 16; ++i) ((uint4 *)blk)[i] = make_uint4(0u, 0u, 0u, 0u);
        for (uint32_t i = 0; i < S; ++i) FREE[i] = (uint16_t)(S - 1 - i);
        memset(&hdr, 0, sizeof hdr);
        const uint32_t cell = M.n_cells ? (gidx / P.replicas_per_cell) % M.n_cells : 0u;
        for (uint32_t i = 0; i < ne; ++i) hs_went_init(&E[i].w, ENTS[i], M, cell, i);
        h_hash = HS_HASH_INIT;
        /* Simulation.__init__: source.start() in order; bootstrap indices come from the global
         * counter (simulation.py:77,145-154), run() restarts the per-heap one at 0. */
        uint64_t boot = 0;
        uint32_t hn = 0;
        for (uint32_t i = 0; i < ne; ++i) {
            if (ENTS[i].kind != HS_ENT_SOURCE) continue;
            hs_went *e = &E[i].w;
            double target = 1.0;
            if (e->i0 == HS_ARR_POISSON && P.trace_arr) {
                if (hdr.np_cursor >= P.n_trace_arr) { hdr.status |= HS_ST_TRACE_EXHAUSTED; break; }
                target = P.trace_arr[(size_t)r * P.n_trace_arr + hdr.np_cursor++]; e->u.src.arr_draws++;
            } else if (e->i0 == HS_ARR_POISSON) {
                target = hs_exp1(hs_uniform(seed, rid, HS_STREAM_ARRIVAL | (i << 8), e->u.src.arr_draws++));
            }
            const int32_t pi = ENTS[i].i3;
            int64_t first;
            if ((FLAGS & HS_WF_PROFILE) && pi > 0) first = hs_next_arrival_profile_ns(&M.profiles[pi - 1], 0, target);
            else first = hs_next_arrival_ns(0, target, e->d0);
            if (first == HS_T_EXHAUSTED) continue;       /* source.start(): RuntimeError, no tick */
            e->u.src.cur_ns = first;
            if (hn >= S) { hdr.status |= HS_ST_FEL_OVERFLOW; break; }
            const uint32_t slot = M.fixed_slots ? i : FREE[S - hn - 1];
            hs_tpay pp; pp.created = 0; pp.aux = 0ull; pp.m0 = HS_EV_SOURCE_TICK | (i << 8); pp.key = -1; pp.hook = 0u; pp.pad = 0u;
            *pay_at(slot) = pp;
            hs_tkey nk; nk.time = first; nk.k2 = (boot++ << 16) | slot;
            uint32_t k = hn++;
            while (k > 0) { const uint32_t p = (k - 1) >> HS_T_SHIFT; const hs_tkey q = kload(p);
                            if (!HS_T_LT(nk.time, nk.k2, q.time, q.k2)) break; kstore(k, q); k = p; }
            kstore(k, nk);
        }
        /* FaultSchedule.start() after the sources and probes (simulation.py:162-169): one Event.once per fault event, its
         * sort index taken from the same global counter (carried in the row); with entity-owned slots the row owns its slot */
        if (FLAGS & HS_WF_FAULTS)
            for (uint32_t i = ne - M.n_faults; i < ne; ++i) {
                if (hn >= S) { hdr.status |= HS_ST_FEL_OVERFLOW; break; }
                const uint32_t slot = M.fixed_slots ? i : FREE[S - hn - 1];
                hs_tpay pp; pp.created = 0; pp.aux = 0ull; pp.m0 = HS_EV_FAULT | (i << 8); pp.key = -1; pp.hook = 0u; pp.pad = 0u;
                *pay_at(slot) = pp;
                hs_tkey nk; nk.time = ENTS[i].l0; nk.k2 = ((uint64_t)(uint32_t)ENTS[i].i3 << 16) | slot;
                uint32_t k = hn++;
                while (k > 0) { const uint32_t p = (k - 1) >> HS_T_SHIFT; const hs_tkey q = kload(p);
                                if (!HS_T_LT(nk.time, nk.k2, q.time, q.k2)) break; kstore(k, q); k = p; }
                kstore(k, nk);
            }
        h_fel = (int32_t)hn;
        hdr.free_top = hn;                               /* free_top holds the heap size in this engine */
        hdr.ctr = 0;
    }

    hs_event_record *rec = (FLAGS & HS_WF_REC) && O.records ? O.records + (size_t)r * P.record_cap : nullptr;
    hs_sink_sample *smp = (FLAGS & HS_WF_REC) && O.samples ? O.samples + (size_t)r * P.sample_cap : nullptr;
    double *svc_out = (FLAGS & HS_WF_REC) && O.service ? O.service + (size_t)r * P.service_cap : nullptr;
    hs_bucket_begin(BK, bacc);

    /* the header's hot fields live in registers for the duration of the launch (the struct itself is addressed through
     * H by the handlers, i.e. it sits in local memory) and are written back with it at the end */
    uint64_t ctr = hdr.ctr;
    int now_n = hdr.now_n;
    uint32_t heap_n = hdr.free_top;
    int64_t top_t = HS_W_EMPTY; uint64_t top_k = ~0ull;  /* the heap's root key, cached */
    if (heap_n) { const hs_tkey t0 = kload(0); top_t = t0.time; top_k = t0.k2; }
    bool paused = false;

    /* ---- phase-locked dispatch ---------------------------------------------------------------------
     * Every replica processes ITS events in exactly the reference's order; what is arranged here is only
     * WHEN a lane runs its next handler.  The loop body is a fixed cycle of phases, one per event kind, in
     * the order the kinds follow each other in the model's same-timestamp chains
     *     heap pop -> TICK | CONTINUATION -> REQ_LB -> ENQUEUE -> SINK ... -> NOTIFY -> LB_RESPONSE -> POLL -> DELIVER -> WORKER
     * and a lane executes a phase only if its next event is of that kind.  After a heap pop all lanes of a
     * warp walk their chains in step, so a phase's code runs once per cycle for all of them (instead of each
     * lane dragging the warp through its own handler: 2.4 of 8 lanes active in round 1's one-switch loop).
     * A lane whose next event is a kind whose phase has passed simply waits for the next cycle. */
    hs_wnow ev; ev.time = 0; ev.idx = 0; ev.created = 0; ev.aux = 0; ev.m0 = 0; ev.key = -1; ev.hook = 0; ev.pad = 0;
    int ev_kind = -1;                                    /* kind of the event held in `ev`, -1: none */
    int64_t prev_t = -1; uint64_t prev_i = ~0ull; uint32_t prev_x = 0u;   /* the previous pop (linked partitions: tie detection) */
    bool alive = true, need_heap = false;

    /* choose the next event: the now tier's minimum unless the heap's root sorts first (then the heap phase pops it) */
    auto next_event = [&]() {
        while (true) {
            ev_kind = -1; need_heap = false;
            const int64_t now0 = h_now;
            if (!(now0 <= P.end_ns) || (hdr.status & (HS_ST_QUEUE_OVERFLOW | HS_ST_FEL_OVERFLOW | HS_ST_TRACE_EXHAUSTED))) { alive = false; return; }
            if (h_processed >= P.max_events) { hdr.status |= HS_ST_EVENT_LIMIT; alive = false; return; }
            int nb = -1; int64_t nt = HS_W_EMPTY; uint64_t ni = ~0ull;
            for (int k = 0; k < now_n; ++k) {
                int64_t t; uint64_t ix; now_key(k, t, ix);
                if (HS_T_LT(t, ix, nt, ni)) { nt = t; ni = ix; nb = k; }
            }
            if (heap_n > 0 && (nb < 0 || HS_T_LT(top_t, top_k >> 16, nt, ni))) {
                if (windowed && top_t > P.window_end_ns) { paused = true; alive = false; return; }
                need_heap = true;
                return;
            }
            if (nb < 0) { alive = false; return; }           /* heap exhausted */
            if (windowed && nt > P.window_end_ns) { paused = true; alive = false; return; }
            ev = now_load(nb);
            if ((FLAGS & HS_WF_LINKED) && M.inbox_cap) {      /* remembered for the tie test at the next heap pop.  An event of
                                                                  * this tier that repeats the key of the delivered event popped just
                                                                  * before it is that event's own child (had it been pending already,
                                                                  * it would have been popped first): no rival, no flag */
                prev_t = ev.time; prev_i = ev.idx; prev_x = 0u;
            }
            now_n--;
            if (nb != now_n) now_store(nb, now_load(now_n));
            h_fel--;
            if (ev.time < now0) continue;                    /* "time travel": skipped (simulation.py:479-489) */
            int k = (int)(ev.m0 & 0xffu);
            if (k == (int)HS_EV_REQ_ANY) {
                const int ek = ENTS[ev.m0 >> 8].kind;
                k = (ek == HS_ENT_SERVER || ek == HS_ENT_CACHE_SERVER) ? HS_EV_REQ_ENQUEUE : ek == HS_ENT_SINK ? HS_EV_REQ_SINK :
                    ek == HS_ENT_COUNTER ? HS_EV_REQ_COUNTER : ek == HS_ENT_PROBE ? HS_EV_PROBE :
                    ek == HS_ENT_SKETCH ? HS_EV_REQ_SKETCH : HS_EV_REQ_LB;
            }
            ev_kind = k;
            return;
        }
    };

    /* insertion of a future event (SourceEvent or ProcessContinuation) into the 4-ary key heap.  (Measured and dropped,
     * round 2: a "lazy" pop that leaves a hole at the root for the chain's first insertion to fill -- heapreplace, one
     * walk instead of two.  It moves the sift-down out of the heap phase, where all lanes of a warp run it together, into
     * the chains, where the tick lanes and the completion lanes each run their own: configs[2] 7.6e9 -> 4.7e9 events/s.) */
    auto heap_slot_store = [&](hs_tkey &fkey, const hs_tpay &fpay, const uint32_t pending) -> bool {   /* the payload goes to its slot at once */
        if (heap_n + pending >= S) { hdr.status |= HS_ST_FEL_OVERFLOW; return false; }
        const uint32_t slot = M.fixed_slots ? (fpay.m0 >> 8) : FREE[S - (heap_n + pending) - 1];   /* entity-owned slot, or the stack's top */
        *pay_at(slot) = fpay;
        fkey.k2 |= slot;
        return true;
    };
    /* an event created during the run that ties with a pending FAULT event (HS_ST_FAULT_TIE) */
    auto fault_tie = [&](const int64_t t, const uint64_t idx) {
        if (hs_fault_tie(ENTS, ne, M.n_faults, t, idx, (const unsigned char *)&E[0].w, (uint32_t)sizeof(hs_tent)))
            hdr.status |= HS_ST_FAULT_TIE;
    };
    auto heap_push_key = [&](const hs_tkey fkey) {                       /* the key sifts up */
        if (FLAGS & HS_WF_FAULTS) fault_tie(fkey.time, fkey.k2 >> 16);
        uint32_t k = heap_n++;
        while (k > 0) {
            const uint32_t p = (k - 1) >> HS_T_SHIFT;
            hs_tkey q;
            if (p == 0) { q.time = top_t; q.k2 = top_k; } else q = kload(p);
            if (!HS_T_LT(fkey.time, fkey.k2, q.time, q.k2)) break;
            kstore(k, q); k = p;
        }
        kstore(k, fkey);
        if (k == 0) { top_t = fkey.time; top_k = fkey.k2; }
        h_fel++;
    };
    auto heap_insert = [&](hs_tkey fkey, const hs_tpay &fpay) {
        if (heap_slot_store(fkey, fpay, 0u)) heap_push_key(fkey);
    };
    /* The fused chains do not sift their (at most two) new keys up themselves: they park them here, and the heap phase
     * inserts them after the tick lanes and the completion lanes of the warp have come together again -- one copy of the
     * sift-up loop, run by all lanes at once, instead of three copies inside the divergent chains. */
    hs_tkey pk0, pk1; pk0.time = pk1.time = 0; pk0.k2 = pk1.k2 = 0ull;
    int n_pk = 0;
    auto chain_insert = [&](hs_tkey fkey, const hs_tpay &fpay) {
        if (!heap_slot_store(fkey, fpay, (uint32_t)n_pk)) return;
        if (n_pk == 0) pk0 = fkey; else pk1 = fkey;
        n_pk++;
    };

    /* ---- fused same-timestamp chains -----------------------------------------------------------------------------
     * The event just popped from the heap (`ev`, a SourceEvent or a ProcessContinuation) starts a chain of events at
     * the same nanosecond: TICK -> [REQ_LB ->] ENQUEUE -> [NOTIFY ->] [LB_RESPONSE ->] [POLL -> DELIVER -> WORKER]
     * or CONTINUATION -> [SINK|COUNTER ->] [POLL -> [DELIVER -> WORKER]].  When nothing else is pending at that
     * nanosecond (empty now tier, the heap's new root strictly later, the events the chain itself schedules strictly
     * later) every event a handler creates is the next pop -- ties among them are resolved by the creation order,
     * which the code below follows index for index, exactly like the lane engine's fused chains -- so the whole
     * chain runs as straight-line code on the entities' state: one load and one store per entity instead of one
     * per event, no now-tier traffic, no per-event dispatch.  Every condition is tested BEFORE anything is
     * changed (draws are pure functions of their index); a chain that does not qualify -- a tie, another topology
     * (tandem, sketch or probe targets), a stop_after source, a full ring, traces, the run / window end, the event
     * limit -- goes through the generic one-event path below, which is the oracle's.  Returns true if it ran.
     * (Measured and dropped, round 2: ONE instruction stream for the tick and the completion lanes where their work is
     * the same -- server-state load, service draw, continuation insert, server-state store -- with the per-kind parts
     * in between, in two orders (the arrival draw after the service draw; the arrival draw between the request for the
     * server's state and its first use).  Fewer warp instructions, but more values live across the shared pieces than 128
     * registers hold (spill reloads sit on the critical path) and more reconvergence points: configs[2] 7.8e9 -> 6.9e9 and
     * 9.0e9 -> 6.8e9 events/s.
     * Also dropped: keeping the second uniform of a Philox block in the entity's spare bytes for the stream's next draw
     * (half of the Philox evaluations) -- the extra live state spills at 128 registers: 8.3e9 -> 7.6e9.) */
    auto emit = [&](const int64_t now, const uint64_t idx, const int kind, const uint32_t ent) {
        if (FLAGS & HS_WF_HASH) h_hash = hs_hash_step(h_hash, now, hs_record_word1(idx, (uint32_t)kind, ent));
        if ((FLAGS & HS_WF_REC) && rec) {
            hs_event_record rc; rc.time_ns = now; rc.sort_index = (uint32_t)idx; rc.kind = (uint8_t)kind;
            rc.pad = 0; rc.entity = (uint16_t)ent;
            rec[hdr.rec_pos] = rc; hdr.rec_pos = (hdr.rec_pos + 1 == P.record_cap) ? 0u : hdr.rec_pos + 1;
        }
        h_processed++;
    };
    /* entity state as six 16-byte vectors: one burst of loads into registers, the dynamic part (vectors 2..5) stored back */
    union went_u { hs_went w; uint4 q[6]; };
    auto went_load = [&](const int i, went_u &x) {
        const uint4 *g = (const uint4 *)&E[i].w;
#pragma unroll
        for (int k = 0; k < 6; ++k) x.q[k] = g[k];
    };
    auto went_store = [&](const int i, const went_u &x) {
        uint4 *g = (uint4 *)&E[i].w;
#pragma unroll
        for (int k = 2; k < 6; ++k) g[k] = x.q[k];
    };
    const bool fuse_on = !P.trace_arr && !P.trace_svc;
    auto fused_chain = [&]() -> bool {
        const int64_t now = ev.time;
        const int k0 = (int)(ev.m0 & 0xffu);
        if (!fuse_on || now_n != 0 || now > P.end_ns || h_processed + 10 > P.max_events) return false;
        if (!(top_t > now)) return false;                       /* the heap's new root must be strictly later */
        const uint32_t ent = ev.m0 >> 8;
        if (k0 == HS_EV_SOURCE_TICK) {
            const hs_entity_desc ds = ENTS[ent];
            if (ds.l0 >= 0 && now > ds.l0) return false;                      /* stop_after reached: no payload */
            const int t1 = ds.target;
            const hs_entity_desc d1 = ENTS[t1];
            went_u xs; went_load((int)ent, xs); hs_went *Xs = &xs.w;
            went_u xl; hs_went *Xl = &xl.w;
            if (d1.kind == HS_ENT_LB) went_load(t1, xl);             /* issued together with the source's: independent lines */
            if ((FLAGS & HS_WF_FAULTS) && (Xs->crashed || (d1.kind == HS_ENT_LB && Xl->crashed))) return false;   /* dropped: generic path */
            const int64_t cur_ns = Xs->u.src.cur_ns; const uint64_t arr_draws = Xs->u.src.arr_draws, key_draws = Xs->u.src.key_draws;
            int32_t key = -1;
            if (ds.i1 > 0) key = hs_routing_key(hs_uniform(seed, rid, HS_STREAM_ROUTING | (ent << 8), key_draws), ds.i1,
                                                ds.i2 > 0 ? M.key_cdf + (ds.i2 - 1) : nullptr);
            int lb = -1, be = t1, slot = 0; uint64_t rr = 0; bool use_rr = false;
            if (d1.kind == HS_ENT_LB) {
                if (d1.i2 <= 0) return false;
                lb = t1;
                if (d1.i0 == HS_LB_KEY_TABLE && key >= 0) slot = M.key_table[key];
                else { rr = Xl->u.lb.rr_index; slot = (int)(rr % (uint64_t)d1.i2); use_rr = true; }
                be = BACKENDS[d1.i1 + slot];
            } else if (d1.kind != HS_ENT_SERVER) return false;
            const hs_entity_desc dv = ENTS[be];
            if (dv.kind != HS_ENT_SERVER) return false;
            went_u xv; went_load(be, xv); hs_went *Xv = &xv.w;       /* requested here, first looked at after the arrival draw below:
                                                                      * the load (a miss, as a rule) has ~200 instructions to arrive */
            /* the next SourceEvent (source.py:166-180) */
            double target = 1.0;
            if (Xs->i0 == HS_ARR_POISSON) target = hs_exp1(hs_uniform(seed, rid, HS_STREAM_ARRIVAL | (ent << 8), arr_draws));
            int64_t nt;
            if ((FLAGS & HS_WF_PROFILE) && ds.i3 > 0) nt = hs_next_arrival_profile_ns(&M.profiles[ds.i3 - 1], cur_ns, target);
            else nt = hs_next_arrival_ns(cur_ns, target, Xs->d0);
            if (nt == HS_T_EXHAUSTED || nt <= now) return false;
            if ((FLAGS & HS_WF_FAULTS) && Xv->crashed) return false;
            const uint32_t q_head = Xv->u.srv.q_head, q_len = Xv->u.srv.q_len; const int32_t active = Xv->u.srv.active;
            const int32_t c_lim = Xv->i0;
            if (q_len >= P.ring) return false;
            const bool was_empty = (q_len == 0);
            const bool drop = (dv.l0 >= 0 && (int64_t)q_len >= dv.l0);
            const bool notify = !drop && was_empty;
            const bool poll = notify && active < c_lim;              /* the worker is idle: POLL -> DELIVER -> WORKER follow */
            /* the service time the WORKER event would draw (server.py:246-253) */
            const uint64_t svc_draws = Xv->u.srv.svc_draws;
            double svc_s = 0.0; int64_t resume_t = 0;
            if (poll) {
                const int64_t dur = (dv.i2 == HS_SVC_EXPONENTIAL)
                    ? hs_seconds_to_ns(HS_DIV(hs_exp1(hs_uniform(seed, rid, HS_STREAM_SERVICE | ((uint32_t)be << 8), svc_draws)), Xv->lambda))
                    : hs_seconds_to_ns(Xv->d0);
                svc_s = hs_ns_to_seconds(dur);
                resume_t = hs_resume_ns(now, svc_s);
                if (resume_t <= now) return false;                   /* a zero-length service resumes at this very nanosecond */
            }
            /* ---- nothing can stop the chain any more: run it ---------------------------------------------------- */
            if (use_rr) {
                /* round robin: the backend of the NEXT request is the next slot, so its state -- the one load of the next
                 * tick chain that depends on another load -- is requested now.  (A key-table balancer's next backend is
                 * known too, the routing key being a pure function of its draw index, but the extra Philox evaluation
                 * cost more than the request saved: configs[3] 2.16e9 -> 2.02e9 events/s at 4 096 replicas.) */
                const int s2 = slot + 1;
                hs_prefetch(&E[BACKENDS[d1.i1 + (s2 == d1.i2 ? 0 : s2)]]);
            }
            h_now = now;
            const uint64_t idxP = ctr, idxT = ctr + 1; ctr += 2;
            emit(now, ev.idx, HS_EV_SOURCE_TICK, ent);
            Xs->u.src.provider++; Xs->u.src.generated++; Xs->u.src.cur_ns = nt;
            if (ds.i1 > 0) Xs->u.src.key_draws = key_draws + 1;
            if (Xs->i0 == HS_ARR_POISSON) Xs->u.src.arr_draws = arr_draws + 1;
            { hs_tkey fk; fk.time = nt; fk.k2 = idxT << 16;
              hs_tpay fp; fp.created = 0; fp.aux = 0ull; fp.m0 = (uint32_t)HS_EV_SOURCE_TICK | (ent << 8); fp.key = -1; fp.hook = 0u; fp.pad = 0u;
              chain_insert(fk, fp); }
            uint64_t idxE = idxP;
            if (lb >= 0) {                                           /* LoadBalancer._forward_request */
                emit(now, idxP, HS_EV_REQ_LB, (uint32_t)lb);
                idxE = ctr++;
            }
            emit(now, idxE, HS_EV_REQ_ENQUEUE, (uint32_t)be);        /* Queue._handle_enqueue */
            uint64_t idxN = 0, idxR = 0;
            if (drop) Xv->u.srv.dropped++;
            else {
                Xv->u.srv.accepted++;
                if (notify) idxN = ctr++;
            }
            if (lb >= 0) idxR = ctr++;                               /* _lb_response hook fires at ENQUEUE time */
            uint64_t idxPoll = 0;
            if (notify) { emit(now, idxN, HS_EV_NOTIFY, (uint32_t)be); if (poll) idxPoll = ctr++; }
            if (lb >= 0) {
                emit(now, idxR, HS_EV_LB_RESPONSE, (uint32_t)lb);    /* in_flight: +1 at forward, -1 here */
                Xl->u.lb.received++; Xl->u.lb.forwarded++; Xl->u.lb.responses++;
                if (use_rr) Xl->u.lb.rr_index = rr + 1;
            }
            if (poll) {
                /* the request is enqueued and polled at once: the ring slot is dead before anyone could read it */
                emit(now, idxPoll, HS_EV_POLL, (uint32_t)be);
                const uint64_t idxD = ctr++;
                emit(now, idxD, HS_EV_DELIVER, (uint32_t)be);
                emit(now, idxE, HS_EV_REQ_WORKER, (uint32_t)be);     /* the payload keeps its own index */
                ctr++;                                               /* inline ProcessContinuation */
                Xv->u.srv.q_head = 0;                                /* the queue is empty again: it restarts at slot 0 (see POLL in hs_handlers.inc) */
                Xv->u.srv.active = active + 1;
                if (dv.i2 == HS_SVC_EXPONENTIAL) Xv->u.srv.svc_draws = svc_draws + 1;
                if ((FLAGS & HS_WF_REC) && svc_out) { svc_out[hdr.svc_pos] = svc_s; hdr.svc_pos = (hdr.svc_pos + 1 == P.service_cap) ? 0u : hdr.svc_pos + 1; }
                hdr.n_svc++;
                const uint64_t idxC = ctr++;
                hs_tkey fk; fk.time = resume_t; fk.k2 = idxC << 16;
                hs_tpay fp; fp.created = now; fp.aux = (uint64_t)__double_as_longlong(svc_s);
                fp.m0 = (uint32_t)HS_EV_CONTINUATION | ((uint32_t)be << 8); fp.key = key; fp.hook = 0x80000000u; fp.pad = 0u;
                chain_insert(fk, fp);
            } else if (!drop) {
                const uint32_t srv_idx = (uint32_t)__double_as_longlong(dv.d1) & 0xffffffu;
                hs_wring_entry *rg = ring0 + (size_t)srv_idx * P.ring;
                hs_wring_entry q; q.created = now; q.idx = idxE; q.key = key;
                if (dv.i1 == HS_Q_PRIORITY) hs_pq_push(rg, q_len, q, (uint32_t)(Xv->u.srv.accepted - 1), M.profile_table + (dv.i3 - 1));
                else rg[(q_head + q_len) & ring_mask] = q;
                Xv->u.srv.q_len = q_len + 1;
            }
            went_store((int)ent, xs);
            if (lb >= 0) went_store(lb, xl);
            went_store(be, xv);
            return true;
        }
        if (k0 == HS_EV_CONTINUATION) {
            const hs_entity_desc dv = ENTS[ent];
            if (dv.kind != HS_ENT_SERVER) return false;               /* e.g. a CachingServer's multi-yield generator */
            const int tgt = dv.target;
            int tkind = 0;
            if (tgt >= 0) { tkind = ENTS[tgt].kind; if (tkind != HS_ENT_SINK && tkind != HS_ENT_COUNTER) return false; }
            if ((FLAGS & HS_WF_FAULTS) && tgt >= 0 && E[tgt].w.crashed) return false;   /* the sink drops the request: generic path */
            went_u xv; went_load((int)ent, xv); hs_went *Xv = &xv.w;
            if (tgt >= 0) hs_prefetch(&E[tgt]);     /* the sink's line: wanted after the draw */
            const uint32_t q_head = Xv->u.srv.q_head, q_len = Xv->u.srv.q_len;
            const int32_t active = Xv->u.srv.active > 0 ? Xv->u.srv.active - 1 : 0;
            const bool poll = (ev.hook & 0x80000000u) && active < Xv->i0;
            const bool start = poll && q_len > 0;
            const uint64_t svc_draws = Xv->u.srv.svc_draws;
            double svc_s = 0.0; int64_t resume_t = 0;
            hs_wring_entry q; q.created = 0; q.idx = 0; q.key = -1;
            if (start) {
                /* the waiting request first: its load (a miss, as a rule) is in flight while the service time is drawn.
                 * A PriorityQueue's root is slot 0 = q_head: the same load; the heap is repaired below */
                const uint32_t srv_idx = (uint32_t)__double_as_longlong(dv.d1) & 0xffffffu;
                const hs_wring_entry *rg = ring0 + (size_t)srv_idx * P.ring;
                q = rg[(dv.i1 == HS_Q_LIFO ? q_head + q_len - 1 : q_head) & ring_mask];
                const int64_t dur = (dv.i2 == HS_SVC_EXPONENTIAL)
                    ? hs_seconds_to_ns(HS_DIV(hs_exp1(hs_uniform(seed, rid, HS_STREAM_SERVICE | (ent << 8), svc_draws)), Xv->lambda))
                    : hs_seconds_to_ns(Xv->d0);
                svc_s = hs_ns_to_seconds(dur);
                resume_t = hs_resume_ns(now, svc_s);
                if (resume_t <= now) return false;
            }
            h_now = now;
            emit(now, ev.idx, HS_EV_CONTINUATION, ent);                /* generator resumes, server.py:255-273 */
            Xv->u.srv.completed++;
            Xv->u.srv.total_service = HS_ADD(Xv->u.srv.total_service, __longlong_as_double((long long)ev.aux));
            uint64_t idxS = 0, idxPoll = 0;
            if (tgt >= 0) idxS = ctr++;
            if (poll) idxPoll = ctr++;
            if (tgt >= 0) {
                went_u xk; went_load(tgt, xk); hs_went *Xk = &xk.w;
                if (tkind == HS_ENT_SINK) {                            /* Sink.handle_event, common.py:36-44 */
                    emit(now, idxS, HS_EV_REQ_SINK, (uint32_t)tgt);
                    const double lat = hs_ns_to_seconds(now - ev.created);
                    if (O.hist) atomicAdd(O.hist + (size_t)r * HS_HIST_BINS + hs_latency_bin(now - ev.created), 1u);
                    double sm = Xk->u.snk.sum, cp = Xk->u.snk.comp;
                    hs_neumaier_add(&sm, &cp, lat);
                    Xk->u.snk.sum = sm; Xk->u.snk.comp = cp;
                    Xk->u.snk.sumsq = HS_ADD(Xk->u.snk.sumsq, HS_MUL(lat, lat));
                    if (lat < Xk->u.snk.mn) Xk->u.snk.mn = lat;
                    if (lat > Xk->u.snk.mx) Xk->u.snk.mx = lat;
                    if (FLAGS & HS_WF_BUCKETS) hs_bucket_add(BK, r, (uint32_t)__double_as_longlong(ENTS[tgt].d1), bacc, now, lat);
                    if ((FLAGS & HS_WF_REC) && smp) { hs_sink_sample qs; qs.completion_ns = now; qs.latency_s = lat; smp[hdr.smp_pos] = qs;
                        hdr.smp_pos = (hdr.smp_pos + 1 == P.sample_cap) ? 0u : hdr.smp_pos + 1; }
                    hdr.n_smp++;
                } else emit(now, idxS, HS_EV_REQ_COUNTER, (uint32_t)tgt);
                Xk->u.snk.received++;
                went_store(tgt, xk);
            }
            int32_t act = active;
            if (poll) {
                emit(now, idxPoll, HS_EV_POLL, ent);                   /* Queue._handle_poll */
                if (start) {
                    const uint64_t idxD = ctr++;
                    emit(now, idxD, HS_EV_DELIVER, ent);
                    emit(now, q.idx, HS_EV_REQ_WORKER, ent);
                    ctr++;                                             /* inline ProcessContinuation */
                    if (dv.i1 == HS_Q_PRIORITY)
                        hs_pq_pop(ring0 + (size_t)((uint32_t)__double_as_longlong(dv.d1) & 0xffffffu) * P.ring, q_len, M.profile_table + (dv.i3 - 1));
                    else Xv->u.srv.q_head = (q_len == 1) ? 0u : (dv.i1 != HS_Q_LIFO ? q_head + 1 : q_head);   /* empty: restart at slot 0 */
                    Xv->u.srv.q_len = q_len - 1;
                    act = active + 1;
                    if (dv.i2 == HS_SVC_EXPONENTIAL) Xv->u.srv.svc_draws = svc_draws + 1;
                    if ((FLAGS & HS_WF_REC) && svc_out) { svc_out[hdr.svc_pos] = svc_s; hdr.svc_pos = (hdr.svc_pos + 1 == P.service_cap) ? 0u : hdr.svc_pos + 1; }
                    hdr.n_svc++;
                    const uint64_t idxC = ctr++;
                    hs_tkey fk; fk.time = resume_t; fk.k2 = idxC << 16;
                    hs_tpay fp; fp.created = q.created; fp.aux = (uint64_t)__double_as_longlong(svc_s);
                    fp.m0 = (uint32_t)HS_EV_CONTINUATION | (ent << 8); fp.key = (int32_t)q.key; fp.hook = 0x80000000u; fp.pad = 0u;
                    chain_insert(fk, fp);
                }
            }
            Xv->u.srv.active = act;
            went_store((int)ent, xv);
            return true;
        }
        return false;
    };

    /* linked partitions: the partition's event router (parallel/routing.py:40-61) -- an event whose target lives in
     * another partition is constructed (its sort index is spent) but never scheduled here: it goes, with the current
     * time, to this replica's outbox, which hs_coordinator_exchange drains at the window barrier */
    auto outbox_send = [&](const uint64_t idx, const int64_t created, const int32_t key, const uint32_t rem, const int64_t now) {
        E[rem].w.u.snk.received++;
        const uint32_t n = O.outbox_n[r];
        if (n >= M.outbox_cap) { hdr.status |= HS_ST_LINK_OVERFLOW; return; }
        hs_xevent x; x.time_ns = now; x.sort_index = idx; x.created_ns = created; x.aux = 0ull; x.key = key; x.ent = (int32_t)rem;
        O.outbox[(size_t)r * M.outbox_cap + n] = x;
        O.outbox_n[r] = n + 1u;
    };

    /* one event: the handler of hs_handlers.inc (kind is warp-uniform at every call site), then the insertion of the
     * (at most one) future event it created */
    auto process = [&](const int kind) {
        const int64_t now = ev.time;
        const uint64_t bi = ev.idx;
        const uint32_t ent = ev.m0 >> 8;
        const int64_t e_created = ev.created;
        const uint64_t e_aux = ev.aux;
        const int32_t e_key = ev.key;
        const uint32_t e_hook = ev.hook;
        /* model row and entity state; handlers work on the copy */
        union { hs_entity_desc d; uint4 q[3]; } du;
        { const uint4 *g = (const uint4 *)&ENTS[ent]; du.q[0] = g[0]; du.q[1] = g[1]; du.q[2] = g[2]; }
        union { hs_went w; uint4 q[6]; } xu;
        { const uint4 *g = (const uint4 *)&E[ent].w;
#pragma unroll
          for (int i = 0; i < 6; ++i) xu.q[i] = g[i]; }
        hs_went *X = &xu.w;
        const uint32_t srv_idx = (uint32_t)__double_as_longlong(du.d.d1) & 0xffffffu;   /* patched in by the host, see hs_model_upload */
        h_now = now;
        if (FLAGS & HS_WF_HASH) h_hash = hs_hash_step(h_hash, now, hs_record_word1(bi, (uint32_t)kind, ent));
        if ((FLAGS & HS_WF_REC) && rec) {
            hs_event_record rc; rc.time_ns = now; rc.sort_index = (uint32_t)bi; rc.kind = (uint8_t)kind;
            rc.pad = 0; rc.entity = (uint16_t)ent;
            rec[hdr.rec_pos] = rc; hdr.rec_pos = (hdr.rec_pos + 1 == P.record_cap) ? 0u : hdr.rec_pos + 1;
        }
        h_processed++;

        bool have_fut = false;                           /* an event creates at most one future event */
        hs_tkey fkey; hs_tpay fpay;
        fkey.time = 0; fkey.k2 = 0ull; fpay.created = 0; fpay.aux = 0ull; fpay.m0 = 0u; fpay.key = -1; fpay.hook = 0u; fpay.pad = 0u;
#define HS_W_PUSH(TIME, IDX, KIND, ENT, CREATED, AUX, KEY, HOOK)                                         \
    do {                                                                                                 \
        const int64_t t_ = (TIME);                                                                       \
        if ((FLAGS & HS_WF_LINKED) && (KIND) == HS_EV_REQ_ANY && M.outbox_cap && ENTS[(ENT)].kind == HS_ENT_REMOTE)                \
            outbox_send((IDX), (CREATED), (KEY), (uint32_t)(ENT), now);                                  \
        else if (t_ <= now) {                                                                                 \
            if (FLAGS & HS_WF_FAULTS) fault_tie(t_, (uint64_t)(IDX));                                    \
            if (now_n >= HS_W_NCAP) hdr.status |= HS_ST_FEL_OVERFLOW;                                    \
            else { hs_wnow n_; n_.time = t_; n_.idx = (IDX); n_.created = (CREATED); n_.aux = (AUX);     \
                   n_.m0 = (uint32_t)(KIND) | ((uint32_t)(ENT) << 8); n_.key = (KEY); n_.hook = (HOOK); n_.pad = 0u; \
                   now_store(now_n++, n_); h_fel++; }                                                \
        } else {                                                                                         \
            if (have_fut) hdr.status |= HS_ST_FEL_OVERFLOW;                                              \
            fkey.time = t_; fkey.k2 = (uint64_t)(IDX) << 16; fpay.created = (CREATED); fpay.aux = (AUX); \
            fpay.m0 = (uint32_t)(KIND) | ((uint32_t)(ENT) << 8); fpay.key = (KEY); fpay.hook = (HOOK);   \
            have_fut = true;                                                                             \
        }                                                                                                \
    } while (0)
#define HS_W_REQ_KIND(TGT) HS_EV_REQ_ANY
#define HS_W_D (du.d)
#define HS_W_SRVIDX srv_idx
#define HS_W_ENT(I) (&E[(I)].w)
#include "hs_handlers.inc"
#undef HS_W_ENT
#undef HS_W_SRVIDX
#undef HS_W_D
#undef HS_W_REQ_KIND
#undef HS_W_PUSH
        /* write the entity's dynamic state back (the union; d0 / lambda / i0 never change) */
        { uint4 *g = (uint4 *)&E[ent].w;
#pragma unroll
          for (int i = 2; i < 6; ++i) g[i] = xu.q[i]; }
        if (have_fut) heap_insert(fkey, fpay);
    };
    /* linked partitions: what the coordinator delivered at the last barrier is scheduled before the first pop
     * (WindowedCoordinator._exchange_events -> Simulation.schedule = heap push, core/simulation.py:195-206); an event
     * that lies behind this replica's clock is dropped by the time-travel test when it is popped.  A delivered event keeps
     * its sender's sort index, so it can tie with a pending FAULT event of this partition: heap_push_key runs the same
     * fault_tie test as for an in-run push (HS_ST_FAULT_TIE).  FAULT rows are pushed at window 0 only (the bootstrap). */
    if ((FLAGS & HS_WF_LINKED) && M.inbox_cap && O.inbox_n) {
        const uint32_t n_in = O.inbox_n[r];
        for (uint32_t k = 0; k < n_in; ++k) {
            const hs_xevent x = O.inbox[(size_t)r * M.inbox_cap + k];
            hs_tkey fk; fk.time = x.time_ns; fk.k2 = x.sort_index << 16;
            hs_tpay fp; fp.created = x.created_ns; fp.aux = 0ull; fp.m0 = (uint32_t)HS_EV_REQ_ANY | ((uint32_t)x.ent << 8);
            fp.key = x.key; fp.hook = 0u; fp.pad = 1u;               /* pad = 1: came over a link (tie detection) */
            heap_insert(fk, fp);
        }
        O.inbox_n[r] = 0u;
    }
    const bool single = (P.lane_stride == 32);          /* one replica per warp: nothing to align, every pass runs the next event */
    next_event();
    while (alive) {
        /* ---- heap phase: the root is the next event (SourceEvent / ProcessContinuation) -------------- */
        if (need_heap) {
            const int64_t now0 = h_now;
            const uint32_t slot = (uint32_t)(top_k & 0xffffu);
            const hs_tpay pp = *pay_at(slot);
            ev.time = top_t; ev.idx = top_k >> 16; ev.created = pp.created; ev.aux = pp.aux;
            ev.m0 = pp.m0; ev.key = pp.key; ev.hook = pp.hook; ev.pad = (FLAGS & HS_WF_LINKED) ? pp.pad : 0u;
            if ((FLAGS & HS_WF_LINKED) && M.inbox_cap) {         /* a delivered event that ties on (time, sort index): see HS_ST_LINK_TIE */
                if (ev.time == prev_t && ev.idx == prev_i && (ev.pad | prev_x)) hdr.status |= HS_ST_LINK_TIE;
                prev_t = ev.time; prev_i = ev.idx; prev_x = ev.pad;
            }
            heap_n--;
            if (!M.fixed_slots) FREE[S - heap_n - 1] = (uint16_t)slot;
            if (heap_n > 0) {                            /* sift-down of the last key from the root */
                const hs_tkey last = kload(heap_n);
                uint32_t k = 0;
                while (true) {
                    const uint32_t c = HS_T_ARITY * k + 1;
                    if (c >= heap_n) break;
                    /* all children at once (one aligned line; the key array has ARITY spare entries, so positions
                     * past the heap's end are readable -- their stale contents are masked out by index) */
                    hs_tkey ch[HS_T_ARITY];
                    if ((FLAGS & HS_WF_HEAPTOP) && c < TOP) {           /* TOP is whole levels: c + j < TOP for all j or for none */
                        const uint4 *b = &Ktop[c * rpb + (uint32_t)tid];
#pragma unroll
                        for (uint32_t j = 0; j < HS_T_ARITY; ++j) {
                            const uint4 q = b[j * rpb];
                            ch[j].time = (int64_t)((uint64_t)q.x | ((uint64_t)q.y << 32)); ch[j].k2 = (uint64_t)q.z | ((uint64_t)q.w << 32);
                        }
                    } else {
#pragma unroll
                        for (uint32_t j = 0; j < HS_T_ARITY; ++j) ch[j] = K[c + j];
                    }
                    hs_tkey best = ch[0]; uint32_t bc = c;
#pragma unroll
                    for (uint32_t j = 1; j < HS_T_ARITY; ++j)
                        if (c + j < heap_n && HS_T_LT(ch[j].time, ch[j].k2, best.time, best.k2)) { best = ch[j]; bc = c + j; }
                    if (!HS_T_LT(best.time, best.k2, last.time, last.k2)) break;
                    kstore(k, best);
                    if (k == 0) { top_t = best.time; top_k = best.k2; }
                    k = bc;
                }
                kstore(k, last);
                if (k == 0) { top_t = last.time; top_k = last.k2; }
                /* the new root is (unless this chain schedules something sooner) the NEXT pop: its payload and, with
                 * entity-owned slots, its entity's state are requested now, a whole chain ahead of their use */
                const uint32_t ns = (uint32_t)(top_k & 0xffffu);
                hs_prefetch(M.fixed_slots ? (const void *)&E[ns] : (const void *)&PAY[ns]);   /* entity-owned slot: ONE line holds both */
            }
            if (heap_n == 0) { top_t = HS_W_EMPTY; top_k = ~0ull; }
            h_fel--;
            need_heap = false;
            int chain_done = 0;
            if ((FLAGS & HS_WF_FAULTS) && (ev.m0 & 0xffu) == HS_EV_FAULT && ENTS[ev.m0 >> 8].i2) {
                E[ev.m0 >> 8].w.u.flt.cancelled++;       /* a cancelled event: counted, not processed (simulation.py:475-477) */
                chain_done = 1;
            }
            else if (ev.time < now0) chain_done = 1;     /* "time travel": skipped (simulation.py:479-489) */
            else if (fused_chain()) chain_done = 1;      /* the whole same-timestamp chain ran as straight-line code */
            else { int k = (int)(ev.m0 & 0xffu);
                   if (k == (int)HS_EV_REQ_ANY) {
                       const int ek = ENTS[ev.m0 >> 8].kind;
                       k = (ek == HS_ENT_SERVER || ek == HS_ENT_CACHE_SERVER) ? HS_EV_REQ_ENQUEUE : ek == HS_ENT_SINK ? HS_EV_REQ_SINK :
                           ek == HS_ENT_COUNTER ? HS_EV_REQ_COUNTER : ek == HS_ENT_PROBE ? HS_EV_PROBE :
                           ek == HS_ENT_SKETCH ? HS_EV_REQ_SKETCH : HS_EV_REQ_LB;
                   }
                   ev_kind = k; }
            asm volatile("" : "+r"(chain_done), "+r"(n_pk));   /* ONE copy of what follows for the tick and the completion lanes, after
                                                                 * they have reconverged (the compiler would otherwise thread it into both chains) */
#pragma unroll 1
            for (int i = 0; i < n_pk; ++i) heap_push_key(i == 0 ? pk0 : pk1);
            n_pk = 0;
            if (chain_done) next_event();
        }
        /* ---- handler phases, in chain order: ONE copy of the handlers (a copy per kind was three times slower when a
         * warp holds a single replica: 170 KB of code); `kind` is warp-uniform in every pass, so the switch inside
         * process() is a uniform branch and the lanes that take it run the same handler.
         * One nibble per pass, low first: TICK 0, CONTINUATION 7, PROBE 11, REQ_LB 1, ENQUEUE 2, SINK 8, COUNTER 10,
         * SKETCH 12, NOTIFY 3, LB_RESPONSE 9, POLL 4, DELIVER 5, WORKER 6 (the HS_EV_* values of include/hs_b200.h), and
         * with HS_WF_FAULTS a last pass for FAULT 13 */
        if (ev_kind < 0) continue;                   /* the fused chain did it all: nothing for the generic passes */
#pragma unroll 1
        for (int ph = 0; ph < ((FLAGS & HS_WF_FAULTS) ? 14 : 13); ++ph) {
            const int kind = single ? ev_kind : (int)((((FLAGS & HS_WF_FAULTS) ? 0xd65493ca821b70ull : 0x65493ca821b70ull) >> (4 * ph)) & 15ull);
            if (alive && ev_kind >= 0 && ev_kind == kind) { process(kind); next_event(); }
        }
    }

    /* ---- publish ------------------------------------------------------------ */
    for (uint32_t i = 0; i < TOP && i < heap_n; ++i) {   /* the shared-memory part of the heap goes back to the resumable image */
        const uint4 q = Ktop[i * rpb + (uint32_t)tid];
        hs_tkey k; k.time = (int64_t)((uint64_t)q.x | ((uint64_t)q.y << 32)); k.k2 = (uint64_t)q.z | ((uint64_t)q.w << 32);
        K[i] = k;
    }
    for (int k = 0; k < now_n && k < HS_T_KS; ++k) {     /* park the shared-memory part of the now tier */
        uint4 *g = (uint4 *)&Ng[k];
        g[0] = Ns[(k * 3 + 0) * rpb + tid];
        g[1] = Ns[(k * 3 + 1) * rpb + tid];
        g[2] = Ns[(k * 3 + 2) * rpb + tid];
    }
    hdr.ctr = ctr; hdr.now_n = now_n; hdr.free_top = heap_n;
    H->now = h_now; H->processed = h_processed; H->hash = h_hash; H->fel_n = h_fel;
    hdr.done = paused ? 0 : 1;
    *Hg = hdr;
    hs_bucket_end(BK, r, bacc);                          /* every row's current time bucket, at the run's end or a pause */
    if (FLAGS & HS_WF_BUCKET_PCT) hdr.status |= hs_bucket_status(BK, r);
    if (O.summaries) {
        hs_replica_summary s;
        s.events_processed = h_processed; s.final_time_ns = h_now;
        s.order_hash = (FLAGS & HS_WF_HASH) ? h_hash : 0ull;
        s.next_sort_index = hdr.ctr; s.n_sink_samples = hdr.n_smp; s.n_service_samples = hdr.n_svc;
        s.heap_left = h_fel; s.status = hdr.status;
        O.summaries[r] = s;
    }
    if (O.stats)
        for (uint32_t i = 0; i < ne; ++i) O.stats[(size_t)r * ne + i] = hs_went_stats_f<FLAGS>(&E[i].w, ENTS[i].kind);
}

/* Two entry points around the one body.  hs_thread_kernel: 128 registers per thread, 8 blocks of 64 threads per SM -- the
 * register file holds 16 warps per SM, which is what an ensemble of thousands of replicas needs to hide its loads; ptxas
 * spills ~130 bytes per thread to get there.  hs_thread_kernel_wide: the same code with the registers it asks for (~208,
 * no spills) at 4 blocks per SM, for launches whose blocks all fit at that occupancy (small ensembles, one replica per
 * warp): every spill reload sits on the one dependent-instruction chain a warp has there.  configs[3] at one GPU's 1 024
 * replicas: 1.125e9 -> 1.25e9 events/s; at 16 384 replicas of configs[2] the wide form would lose a quarter (second wave).
 * Both take the bucket arguments last, as the lane and warp kernels do: hs_bucket_args with HS_WF_BUCKETS,
 * hs_bucket_pct_args with HS_WF_BUCKET_PCT, the empty hs_no_bucket_args otherwise. */
template <int FLAGS>
__global__ void __launch_bounds__(HS_THREAD_BLOCK, HS_T_MINBLOCKS)
hs_thread_kernel(hs_warp_model M, hs_kernel_run P, unsigned char *__restrict__ blocks,
                 hs_wring_entry *__restrict__ rings, hs_kernel_out O,
                 typename hs_bucket_args_of<(FLAGS & HS_WF_BUCKETS) != 0, (FLAGS & HS_WF_BUCKET_PCT) != 0>::type BK)
{
    hs_thread_body<FLAGS>(M, P, blocks, rings, O, BK);
}

#define HS_T_WIDE_BLOCKS 4
template <int FLAGS>
__global__ void __launch_bounds__(HS_THREAD_BLOCK, HS_T_WIDE_BLOCKS)
hs_thread_kernel_wide(hs_warp_model M, hs_kernel_run P, unsigned char *__restrict__ blocks,
                      hs_wring_entry *__restrict__ rings, hs_kernel_out O,
                      typename hs_bucket_args_of<(FLAGS & HS_WF_BUCKETS) != 0, (FLAGS & HS_WF_BUCKET_PCT) != 0>::type BK)
{
    hs_thread_body<FLAGS>(M, P, blocks, rings, O, BK);
}

/* The flag words each entry point is built for (hs_engine.cu launches through a table of them): the general engines'
 * set, and the wide kernel never with HS_WF_HEAPTOP (it is for launches without a heap top) or HS_WF_LINKED (linked
 * launches never take it). */
constexpr bool hs_thread_built(int F) { return hs_general_built(F); }
constexpr bool hs_thread_wide_built(int F) { return hs_general_built(F) && !(F & (HS_WF_HEAPTOP | HS_WF_LINKED)); }

#endif /* HS_THREAD_ENGINE_CUH */
