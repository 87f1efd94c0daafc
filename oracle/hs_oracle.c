/* hs_oracle.c -- CPU restatement of the reference's Simulation.run() hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (happy-simulator_b200/,
 * include/) may import, link or execute this file; only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do,
 * and only as the checker.  The product path is the CUDA engine and fails
 * loudly without it.
 *
 * Parity pinning: this restatement is checked, event by event, against the
 * UNMODIFIED reference (imported from /root/reference, driven through its own
 * LatencyDistribution / ArrivalTimeProvider plug-in points by the Philox
 * sampler of happy-simulator_b200/csrc/hs_sampler.h) by
 * tests/golden/gen_golden.py; the fixtures it wrote are committed under
 * tests/golden/ and tests/test_oracle_golden.py replays them.  The reference's
 * own deterministic known answers for this path (SURVEY.md section 4) are
 * restated in tests/test_oracle_golden.py (README quick-start, counter KAT, the
 * stock-seed runs), tests/test_sampler.py (arrival-time regression vectors) and
 * tests/test_sketch_kats.py (the sketch classes' answers on fixed streams).
 *
 * The structure follows the reference one to one (paths under /root/reference):
 *   run loop            happysimulator/core/simulation.py:449-505 (_execute_until)
 *   heap                happysimulator/core/event_heap.py:54-113 + CPython heapq
 *   order key           happysimulator/core/event.py:337-344 (time, _sort_index)
 *   creation counters   happysimulator/core/event.py:53-77, event_heap.py:48,
 *                       core/sim_future.py:64-73 (global at bootstrap, per heap in run)
 *   completion hooks    happysimulator/core/event.py:277-311
 *   generators          happysimulator/core/event.py:313-325,465-533
 *   Source              happysimulator/load/source.py:67-86,120-180
 *   arrival providers   happysimulator/load/arrival_time_provider.py:57-82
 *   Queue/Driver/Worker happysimulator/components/queue.py:115-166,
 *                       queue_driver.py:57-99, queued_resource.py:38-49,138-143
 *   Server              happysimulator/components/server/server.py:202-273,
 *                       server/concurrency.py:66-140
 *   Sink / Counter      happysimulator/components/common.py:36-44,92-95
 *   LoadBalancer        happysimulator/components/load_balancer/load_balancer.py:347-473,
 *                       strategies.py:61-68 (RoundRobin), :411-433 (ConsistentHash.select,
 *                       as a host-precomputed key -> backend table)
 *   SketchCollector     happysimulator/components/sketching/sketch_collector.py:79-98 over
 *                       sketching/hyperloglog.py:137-165 / count_min_sketch.py:168-187 (add), with the
 *                       per-key SHA-256 results precomputed on the host (csrc/hs_sketch.h)
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <math.h>

#include "../include/hs_b200.h"
#include "../happy-simulator_b200/csrc/hs_sampler.h"
#include "../happy-simulator_b200/csrc/hs_profile.h"
#include "../happy-simulator_b200/csrc/hs_sketch.h"

/* ---- one pending Event object ------------------------------------------ */
typedef struct oev {
    int64_t time;        /* Event.time (ns)                                       */
    uint64_t idx;        /* Event._sort_index                                     */
    int32_t kind;        /* HS_EV_*                                               */
    int32_t ent;         /* target entity id                                      */
    /* request context (Event.context): shared by forward()/LB copies            */
    int64_t created_at;  /* context["created_at"]                                 */
    uint32_t req_id;     /* context["request_id"]                                 */
    int32_t key;         /* context["metadata"]["client_id"], -1 if none          */
    int32_t lb_hook;     /* LoadBalancer on_complete hook: LB entity id, -1 none  */
    int32_t poll_hook;   /* QueueDriver schedule_poll hook: server id, -1 none    */
    double svc_s;        /* CONTINUATION: the service time the generator yielded  */
    int32_t stage;       /* CONTINUATION at a CachingServer: which yield resumes (1, 2, 3) | was_in_cache << 8 */
    uint64_t payload_idx;/* DELIVER: _sort_index of the payload Event it carries  */
#ifdef HS_ORACLE_HIGH_WATER
    int32_t hw_future;   /* scheduled strictly later than its creation, or at the bootstrap / a barrier */
#endif
} oev;

/* ---- CPython heapq (Lib/heapq.py: heappush/_siftdown, heappop/_siftup) -- */
#ifdef HS_ORACLE_HIGH_WATER
/* High-water marks of the structures the device bounds, kept only in the instrumented build (-DHS_ORACLE_HIGH_WATER,
 * tests/high_water_lib.py).  The reference's heap has no limit; on the device an event created at or before the
 * clock joins the same-timestamp ("now") tier (HS_W_PUSH: t <= now) and every other event takes a future-event slot,
 * as do the bootstrap events and what a barrier delivers.  One row of HS_HW_FIELDS + n_entities counters per replica:
 *   HS_HW_NOW       most now-tier events pending at once (the event being handled is not pending)
 *   HS_HW_NOW_POP   most now-tier events pending when a future event is popped (the warp engine moves that event
 *                   into its now tier before handling it, so it needs a free entry then)
 *   HS_HW_FUTURE    most future events pending at once
 *   HS_HW_OUTBOX    linked runs: most cross-partition sends in one window, the ones the full outbox dropped included
 *   HS_HW_INBOX     linked runs: most events delivered into this partition at one barrier
 *   HS_HW_FIELDS+i  entity i: the longest its queue was right after an enqueue (a bounded queue drops first) */
enum { HS_HW_NOW, HS_HW_NOW_POP, HS_HW_FUTURE, HS_HW_OUTBOX, HS_HW_INBOX, HS_HW_FIELDS };
typedef struct { oev *a; size_t n, cap;
                 int64_t clock;            /* time of the event being handled; INT64_MIN at the bootstrap and a barrier */
                 uint32_t n_now, n_future, hw[HS_HW_FIELDS]; } oheap;
#define HS_HW_MAX(x, v) do { if ((v) > (x)) (x) = (v); } while (0)
#else
typedef struct { oev *a; size_t n, cap; } oheap;
#endif

static int ev_lt(const oev *x, const oev *y)    /* Event.__lt__, event.py:337-344 */
{
    if (x->time != y->time) return x->time < y->time;
    return x->idx < y->idx;
}

static void heap_siftdown(oheap *h, size_t start, size_t pos)
{
    oev item = h->a[pos];
    while (pos > start) {
        size_t parent = (pos - 1) >> 1;
        if (ev_lt(&item, &h->a[parent])) { h->a[pos] = h->a[parent]; pos = parent; continue; }
        break;
    }
    h->a[pos] = item;
}

static void heap_siftup(oheap *h, size_t pos)
{
    size_t end = h->n, start = pos;
    oev item = h->a[pos];
    size_t child = 2 * pos + 1;
    while (child < end) {
        size_t right = child + 1;
        if (right < end && !ev_lt(&h->a[child], &h->a[right])) child = right;
        h->a[pos] = h->a[child];
        pos = child;
        child = 2 * pos + 1;
    }
    h->a[pos] = item;
    heap_siftdown(h, start, pos);
}

static void heap_push(oheap *h, const oev *e)
{
    if (h->n == h->cap) {
        h->cap = h->cap ? h->cap * 2 : 64;
        h->a = (oev *)realloc(h->a, h->cap * sizeof(oev));
    }
    h->a[h->n++] = *e;
#ifdef HS_ORACLE_HIGH_WATER
    if ((h->a[h->n - 1].hw_future = e->time > h->clock)) { h->n_future++; HS_HW_MAX(h->hw[HS_HW_FUTURE], h->n_future); }
    else { h->n_now++; HS_HW_MAX(h->hw[HS_HW_NOW], h->n_now); }
#endif
    heap_siftdown(h, 0, h->n - 1);
}

static oev heap_pop(oheap *h)
{
    oev last = h->a[--h->n];
    if (h->n) { oev ret = h->a[0]; h->a[0] = last; heap_siftup(h, 0); return ret; }
    return last;
}

/* ---- entity state ------------------------------------------------------ */
typedef struct { int64_t created_at; uint64_t idx; uint32_t req_id; int32_t key; } oreq;

typedef struct oent {
    hs_entity_desc d;        /* with the cell override applied                    */
    /* SOURCE */
    int64_t cur_ns;          /* ArrivalTimeProvider.current_time                  */
    uint64_t arr_draws;      /* arrival draws consumed                            */
    uint64_t key_draws;      /* routing-key draws consumed                        */
    int64_t generated_count; /* Source._generated_count                           */
    int64_t provider_count;  /* SimpleEventProvider._generated                    */
    /* SERVER */
    oreq *q; size_t q_head, q_len, q_cap;   /* FIFOQueue / LIFOQueue deque        */
    int32_t active;          /* FixedConcurrency._active                          */
    uint64_t svc_draws;
    double lambda;           /* ExponentialLatency._lambda = 1 / mean             */
    int64_t accepted, dropped, completed, rejected;
    double total_service;    /* Server._total_service_time                        */
    /* SINK / COUNTER */
    int64_t received;
    double sum, comp, sumsq, mn, mx;   /* sum/comp: Neumaier state of sum(latencies_s) */
    /* LB */
    uint64_t rr_index;       /* RoundRobin._index                                 */
    int64_t lb_received, lb_forwarded, lb_in_flight, lb_responses;
    uint32_t lb_next_request_id;
    /* SKETCH */
    int64_t sk_processed, sk_added;   /* SketchCollector._events_processed, sketch._total_count */
    /* CACHE_SERVER */
    double *cache_ins;                /* TTLEviction._insert_times per key slot (seconds; 0 = not cached)    */
    int64_t cache_hits, cache_misses, cache_size;
    int cache_own;                    /* cache_ins is a private allocation (no hs_outputs.sketches buffer)   */
    uint8_t *sk_state;                /* this replica's registers / counters (in hs_outputs.sketches) */
#ifdef HS_ORACLE_HIGH_WATER
    uint32_t hw_queue;                /* longest queue right after an enqueue                                */
#endif
} oent;

typedef struct orun {
    const hs_model_desc *m;
    const hs_run_params *p;
    oent *ents;
    oheap heap;
    uint64_t counter;        /* active creation counter                           */
    uint64_t seed; uint32_t rid;
    int64_t now;
    uint32_t status;
    /* optional externally supplied draws (hs_oracle_run_trace): the reference's own
     * RNG outputs, so the restatement can be checked against a STOCK-seed run */
    const double *trace_targets; uint64_t n_trace_targets;   /* -log(1-U) per arrival  */
    const double *trace_service; uint64_t n_trace_service;   /* -log(1-U) of random.random() */
    uint64_t np_cursor, py_cursor;   /* the process-global streams are shared by all consumers */
    /* outputs of this replica */
    hs_event_record *rec;
    hs_sink_sample *smp; int64_t n_smp;
    uint32_t *hist;
    double *svc; int64_t n_svc;
    int64_t processed; uint64_t hash;     /* events processed so far, running order hash               */
    /* linked partitions: this partition's outbox (routing.py:17-63), drained by the coordinator at every barrier */
    hs_xevent *outbox; uint32_t outbox_n, outbox_cap;
    uint32_t r;                           /* replica slot in the outputs                                */
    const hs_outputs *out;
#ifdef HS_ORACLE_HIGH_WATER
    uint32_t hw_sent, hw_received;        /* cross-partition sends / deliveries in the current window   */
#endif
} orun;

static void q_push(oent *s, const oreq *r)
{
    if (s->q_len == s->q_cap) {
        size_t ncap = s->q_cap ? s->q_cap * 2 : 16;
        oreq *nq = (oreq *)malloc(ncap * sizeof(oreq));
        for (size_t i = 0; i < s->q_len; ++i) nq[i] = s->q[(s->q_head + i) % s->q_cap];
        free(s->q); s->q = nq; s->q_cap = ncap; s->q_head = 0;
    }
    s->q[(s->q_head + s->q_len) % s->q_cap] = *r;
    s->q_len++;
}

static oreq q_pop(oent *s)
{
    oreq r;
    if (s->d.i1 == HS_Q_LIFO) {          /* LIFOQueue.pop: deque.pop() (right)   */
        r = s->q[(s->q_head + s->q_len - 1) % s->q_cap];
    } else {                              /* FIFOQueue.pop: deque.popleft()       */
        r = s->q[s->q_head];
        s->q_head = (s->q_head + 1) % s->q_cap;
    }
    s->q_len--;
    return r;
}

static oev new_event(orun *R, int64_t time, int kind, int ent)   /* Event.__init__ */
{
    oev e; memset(&e, 0, sizeof e);
    e.time = time; e.kind = kind; e.ent = ent;
    e.idx = R->counter++;                 /* _next_sort_index(), event.py:62-67   */
    e.key = -1; e.lb_hook = -1; e.poll_hook = -1;
    return e;
}

static int request_kind_for(const orun *R, int ent)
{
    switch (R->ents[ent].d.kind) {
    case HS_ENT_SERVER: case HS_ENT_CACHE_SERVER: return HS_EV_REQ_ENQUEUE;
    case HS_ENT_SINK: return HS_EV_REQ_SINK;
    case HS_ENT_COUNTER: return HS_EV_REQ_COUNTER;
    case HS_ENT_LB: return HS_EV_REQ_LB;
    case HS_ENT_PROBE: return HS_EV_PROBE;
    case HS_ENT_SKETCH: return HS_EV_REQ_SKETCH;
    default: return -1;
    }
}

/* ArrivalTimeProvider.next_arrival_time, constant-rate fast path
 * (arrival_time_provider.py:66-82). */
static int64_t next_arrival(orun *R, int sid, oent *s)
{
    double target;
    if (s->d.i0 == HS_ARR_POISSON && R->trace_targets) {
        target = R->np_cursor < R->n_trace_targets ? R->trace_targets[R->np_cursor] : 1e300;
        R->np_cursor++; s->arr_draws++;
    } else if (s->d.i0 == HS_ARR_POISSON) {
        double u = hs_uniform(R->seed, R->rid, HS_STREAM_ARRIVAL | ((uint32_t)sid << 8), s->arr_draws++);
        target = hs_exp1(u);              /* poisson_arrival.py:31                */
    } else {
        target = 1.0;                     /* constant_arrival.py:21-23            */
    }
    if (s->d.i3 > 0) {                    /* non-constant profile: Simpson + Brent path */
        int64_t t = hs_next_arrival_profile_ns(&R->m->profiles[s->d.i3 - 1], s->cur_ns, target);
        if (t != HS_T_EXHAUSTED) s->cur_ns = t;
        return t;
    }
    s->cur_ns = hs_next_arrival_ns(s->cur_ns, target, s->d.d0);
    return s->cur_ns;
}

/* QueueDriver._handle_work_payload.schedule_poll (queue_driver.py:79-85). */
static void run_poll_hook(orun *R, int server)
{
    oent *s = &R->ents[server];
    if (s->d.kind == HS_ENT_CACHE_SERVER || s->active < s->d.i0) {   /* target.has_capacity(); Entity's default is True */
        oev p = new_event(R, R->now, HS_EV_POLL, server);
        heap_push(&R->heap, &p);
    }
}

/* Event._run_completion_hooks for a request whose non-generator handler just
 * returned (event.py:277-283): only the LoadBalancer on_complete hook can be
 * attached at that point (load_balancer.py:414-427). */
static void run_request_hooks(orun *R, oev *e)
{
    if (e->lb_hook >= 0) {
        oev r = new_event(R, R->now, HS_EV_LB_RESPONSE, e->lb_hook);
        heap_push(&R->heap, &r);
        e->lb_hook = -1;                  /* on_complete.clear()                  */
    }
}

static void handle(orun *R, oev *e)
{
    oent *E = &R->ents[e->ent];
    switch (e->kind) {
    case HS_EV_SOURCE_TICK: {             /* Source.handle_event, source.py:142-180 */
        int have_payload = 0; oev pay;
        if (!(E->d.l0 >= 0 && R->now > E->d.l0)) {   /* stop_after, source.py:68 */
            E->provider_count++;
            pay = new_event(R, R->now, request_kind_for(R, E->d.target), E->d.target);
            pay.created_at = R->now;
            pay.req_id = (uint32_t)E->provider_count;
            if (E->d.i1 > 0) {            /* routing key: client_id ~ Uniform{0..pop-1} or Zipf (zipf.py:112-123) */
                double u = hs_uniform(R->seed, R->rid, HS_STREAM_ROUTING | ((uint32_t)e->ent << 8), E->key_draws++);
                pay.key = hs_routing_key(u, E->d.i1, E->d.i2 > 0 ? R->m->key_cdf + (E->d.i2 - 1) : NULL);
            }
            have_payload = 1;
        }
        E->generated_count++;
        int64_t nt = next_arrival(R, e->ent, E);
        if (have_payload) heap_push(&R->heap, &pay);
        if (nt != HS_T_EXHAUSTED) {       /* RuntimeError: "Source exhausted", source.py:176-180 */
            oev tick = new_event(R, nt, HS_EV_SOURCE_TICK, e->ent);
            heap_push(&R->heap, &tick);
        }
        break;
    }
    case HS_EV_REQ_LB: {                  /* LoadBalancer._forward_request, :347-433 */
        E->lb_received++;
        int nb = E->d.i2;
        if (nb <= 0) break;               /* no healthy backends -> rejected     */
        int slot;
        if (E->d.i0 == HS_LB_KEY_TABLE && e->key >= 0)
            slot = R->m->key_table[e->key];                 /* ConsistentHash.select    */
        else { slot = (int)(E->rr_index % (uint64_t)nb); E->rr_index++; } /* RoundRobin  */
        int backend = R->m->backends[E->d.i1 + slot];
        E->lb_next_request_id++;
        E->lb_in_flight++;
        E->lb_forwarded++;
        oev f = new_event(R, R->now, request_kind_for(R, backend), backend);
        f.created_at = e->created_at; f.req_id = e->req_id; f.key = e->key;
        f.lb_hook = e->ent;
        heap_push(&R->heap, &f);
        run_request_hooks(R, e);          /* hooks of the original (none from a Source) */
        break;
    }
    case HS_EV_REQ_ENQUEUE: {             /* Queue._handle_enqueue, queue.py:122-147 */
        int was_empty = (E->q_len == 0);
        const int64_t qcap = E->d.kind == HS_ENT_CACHE_SERVER ? -1 : E->d.l0;   /* CachingServer: FIFOQueue(), unbounded */
        int accepted = !(qcap >= 0 && (int64_t)E->q_len >= qcap);        /* queue_policy.py:94-98 */
        if (!accepted) {
            E->dropped++;
        } else {
            oreq r; r.created_at = e->created_at; r.idx = e->idx; r.req_id = e->req_id; r.key = e->key;
            q_push(E, &r);
#ifdef HS_ORACLE_HIGH_WATER
            HS_HW_MAX(E->hw_queue, (uint32_t)E->q_len);
#endif
            E->accepted++;
            if (was_empty) {
                oev n = new_event(R, R->now, HS_EV_NOTIFY, e->ent);
                heap_push(&R->heap, &n);
            }
        }
        run_request_hooks(R, e);          /* _lb_response fires at ENQUEUE time  */
        break;
    }
    case HS_EV_NOTIFY:                    /* QueueDriver._handle_notify, :92-99  */
        if (E->d.kind == HS_ENT_CACHE_SERVER || E->active < E->d.i0) {
            oev p = new_event(R, R->now, HS_EV_POLL, e->ent);
            heap_push(&R->heap, &p);
        }
        break;
    case HS_EV_POLL:                      /* Queue._handle_poll, queue.py:149-166 */
        if (E->q_len > 0) {
            oreq r = q_pop(E);
            oev d = new_event(R, R->now, HS_EV_DELIVER, e->ent);
            d.created_at = r.created_at; d.req_id = r.req_id; d.key = r.key;
            d.payload_idx = r.idx;       /* QueueDeliverEvent.payload is the queued Event object */
            heap_push(&R->heap, &d);
        }
        break;
    case HS_EV_DELIVER: {                 /* _handle_work_payload, queue_driver.py:78-90 */
        oev w; memset(&w, 0, sizeof w);
        w.time = R->now; w.kind = HS_EV_REQ_WORKER; w.ent = e->ent;
        w.idx = e->payload_idx;           /* the payload keeps its OLD _sort_index */
        w.created_at = e->created_at; w.req_id = e->req_id; w.key = e->key;
        w.lb_hook = -1; w.poll_hook = e->ent;
        heap_push(&R->heap, &w);
        break;
    }
    case HS_EV_REQ_WORKER: {              /* Server.handle_queued_event first step */
        R->counter++;                     /* inline ProcessContinuation, event.py:314-325 */
        if (E->d.kind == HS_ENT_CACHE_SERVER) {
            /* CachingServer.handle_queued_event up to its first yield (examples/load-balancing/common.py:197-213):
             * was_in_cache = key in cache and not TTLEviction.is_expired(key) (eviction_policies.py:215-226, clock =
             * self.now.to_seconds()); then `yield cache_read_latency_s` -> ProcessContinuation at now + int(delay * 1e9) */
            E->active++;
            const int slot = e->key >= 0 && e->key < E->d.i0 ? e->key : E->d.i0;       /* no customer id: "unknown" */
            const double ins = E->cache_ins[slot];
            const int was_in = ins != 0.0 && !(hs_ns_to_seconds(R->now) - ins >= E->d.d0);
            oev c = new_event(R, R->now + (int64_t)E->d.i2, HS_EV_CONTINUATION, e->ent);
            c.created_at = e->created_at; c.req_id = e->req_id; c.key = e->key;
            c.poll_hook = e->poll_hook; c.stage = 1 | (was_in << 8);
            heap_push(&R->heap, &c);
            break;
        }
        if (E->active >= E->d.i0) {       /* acquire failed, server.py:223-234   */
            E->rejected++;
            R->status |= HS_ST_REJECT_PATH;
            run_poll_hook(R, e->ent);     /* StopIteration -> hooks, event.py:522-533 */
            break;
        }
        E->active++;
        int64_t dur_ns;
        if (E->d.i2 == HS_SVC_EXPONENTIAL && R->trace_service) {
            /* random.expovariate(lambd) = -log(1.0 - random()) / lambd; the trace holds -log(1 - U) */
            double sample = (R->py_cursor < R->n_trace_service ? R->trace_service[R->py_cursor] : 1e300) / E->lambda;
            R->py_cursor++; E->svc_draws++;
            dur_ns = hs_seconds_to_ns(sample);            /* Duration.from_seconds(sample) */
        } else if (E->d.i2 == HS_SVC_EXPONENTIAL) {
            double u = hs_uniform(R->seed, R->rid, HS_STREAM_SERVICE | ((uint32_t)e->ent << 8), E->svc_draws++);
            dur_ns = hs_exp_latency_ns(u, E->lambda);     /* exponential.py:41-45 */
        } else {
            dur_ns = hs_seconds_to_ns(E->d.d0);           /* constant.py:33-35    */
        }
        double service_time_s = hs_ns_to_seconds(dur_ns); /* server.py:246-247    */
        if (R->svc && R->p->service_cap) R->svc[R->n_svc % R->p->service_cap] = service_time_s;
        R->n_svc++;
        oev c = new_event(R, hs_resume_ns(R->now, service_time_s), HS_EV_CONTINUATION, e->ent);
        c.created_at = e->created_at; c.req_id = e->req_id; c.key = e->key;
        c.poll_hook = e->poll_hook; c.svc_s = service_time_s;
        heap_push(&R->heap, &c);
        break;
    }
    case HS_EV_CONTINUATION: {            /* generator resumes, server.py:255-273 */
        if (E->d.kind == HS_ENT_CACHE_SERVER) {               /* common.py:215-232 */
            const int stage = e->stage & 0xff, was_in = (e->stage >> 8) & 1;
            const int slot = e->key >= 0 && e->key < E->d.i0 ? e->key : E->d.i0;
            int next_stage = 0; int64_t delay = 0;
            if (stage == 1) {
                if (was_in) { E->cache_hits++; next_stage = 3; delay = (int64_t)E->d.i3; }     /* on_access: TTL ignores it */
                else { E->cache_misses++; next_stage = 2; delay = E->d.l0; }                  /* yield datastore latency  */
            } else if (stage == 2) {          /* _populate_cache: cache[key] = value; on_insert(key) records the time */
                if (E->cache_ins[slot] == 0.0) E->cache_size++;
                E->cache_ins[slot] = hs_ns_to_seconds(R->now);
                next_stage = 3; delay = (int64_t)E->d.i3;
            } else {                          /* requests_processed += 1; return [] -> completion hooks */
                E->completed++;
                E->active = E->active > 0 ? E->active - 1 : 0;
                if (e->poll_hook >= 0) run_poll_hook(R, e->poll_hook);
                break;
            }
            oev c = new_event(R, R->now + delay, HS_EV_CONTINUATION, e->ent);
            c.created_at = e->created_at; c.req_id = e->req_id; c.key = e->key;
            c.poll_hook = e->poll_hook; c.stage = next_stage;
            heap_push(&R->heap, &c);
            break;
        }
        E->active = E->active > 0 ? E->active - 1 : 0;    /* FixedConcurrency.release */
        E->completed++;
        E->total_service += e->svc_s;
        if (E->d.target >= 0) {           /* Entity.forward, entity.py:83-105     */
            oev f = new_event(R, R->now, request_kind_for(R, E->d.target), E->d.target);
            f.created_at = e->created_at; f.req_id = e->req_id; f.key = e->key;
            if (R->ents[E->d.target].d.kind == HS_ENT_REMOTE) {
                /* the partition's event router (routing.py:40-61): a target outside this partition -> the event,
                 * already constructed (its sort index is spent), goes to the outbox with the current time */
                R->ents[E->d.target].received++;
#ifdef HS_ORACLE_HIGH_WATER
                R->hw_sent++; HS_HW_MAX(R->heap.hw[HS_HW_OUTBOX], R->hw_sent);
#endif
                if (R->outbox_n < R->outbox_cap) {
                    hs_xevent *x = &R->outbox[R->outbox_n++];
                    x->time_ns = R->now; x->sort_index = f.idx; x->created_ns = f.created_at; x->aux = 0;
                    x->key = f.key; x->ent = E->d.target;
                } else R->status |= HS_ST_LINK_OVERFLOW;
            } else heap_push(&R->heap, &f);
        }
        if (e->poll_hook >= 0) run_poll_hook(R, e->poll_hook);
        break;
    }
    case HS_EV_REQ_SINK: {                /* Sink.handle_event, common.py:36-44   */
        E->received++;
        double lat = hs_ns_to_seconds(R->now - e->created_at);
        if (R->hist) R->hist[hs_latency_bin(R->now - e->created_at)]++;
        hs_neumaier_add(&E->sum, &E->comp, lat); E->sumsq += lat * lat;
        if (lat < E->mn) E->mn = lat;
        if (lat > E->mx) E->mx = lat;
        if (R->smp && R->p->sample_cap) {
            hs_sink_sample *q = &R->smp[R->n_smp % R->p->sample_cap];
            q->completion_ns = R->now; q->latency_s = lat;
        }
        R->n_smp++;
        run_request_hooks(R, e);
        break;
    }
    case HS_EV_PROBE: {                   /* measure_callback, instrumentation/probe.py:51-66 */
        const oent *T = &R->ents[E->d.target];
        double val = 0.0;
        switch (E->d.i0) {                /* getattr(target, metric) */
        case HS_METRIC_DEPTH: val = (double)T->q_len; break;                       /* queued_resource.py:113 */
        case HS_METRIC_ACTIVE_REQUESTS: val = (double)T->active; break;            /* server.py:154 */
        case HS_METRIC_UTILIZATION: val = T->d.i0 == 0 ? 0.0 : (double)T->active / (double)T->d.i0; break;  /* server.py:164-173 */
        case HS_METRIC_AVAILABLE_CAPACITY: val = (double)(T->d.i0 - T->active); break;
        case HS_METRIC_STATS_ACCEPTED: val = (double)T->accepted; break;
        case HS_METRIC_STATS_DROPPED: val = (double)T->dropped; break;
        case HS_METRIC_EVENTS_RECEIVED: case HS_METRIC_TOTAL: val = (double)T->received; break;
        case HS_METRIC_GENERATED_COUNT: val = (double)T->generated_count; break;
        }
        E->received++;
        hs_neumaier_add(&E->sum, &E->comp, val);
        if (val < E->mn) E->mn = val;
        if (val > E->mx) E->mx = val;
        if (R->smp && R->p->sample_cap) {
            hs_sink_sample *q = &R->smp[R->n_smp % R->p->sample_cap];
            q->completion_ns = R->now; q->latency_s = val;
        }
        R->n_smp++;
        break;
    }
    case HS_EV_REQ_COUNTER:               /* Counter.handle_event, common.py:92-95 */
        E->received++;
        run_request_hooks(R, e);
        break;
    case HS_EV_REQ_SKETCH:                /* SketchCollector.handle_event, sketch_collector.py:79-98 */
        if (E->d.i0 == HS_SK_TDIGEST) {   /* QuantileEstimator (quantile_estimator.py:96-110): value = latency in s */
            if (E->sk_state && !hs_tdigest_add(E->sk_state, E->d.d0, (uint32_t)E->d.i2, (uint32_t)E->d.i3,
                                               hs_ns_to_seconds(R->now - e->created_at)))
                R->status |= HS_ST_SKETCH_OVERFLOW;
            E->sk_added++;
        } else if (e->key >= 0) {         /* value is not None: sketch.add(value) */
            if (E->sk_state)
                hs_sketch_add(E->sk_state, R->m->sketch_tables + E->d.i1, E->d.i0, E->d.i2, E->d.i3, E->d.l0, e->key);
            E->sk_added++;
        }
        E->sk_processed++;
        run_request_hooks(R, e);
        break;
    case HS_EV_LB_RESPONSE:               /* LoadBalancer._handle_response, :435-473 */
        if (E->lb_in_flight > 0) E->lb_in_flight--;
        E->lb_responses++;
        break;
    default: break;
    }
}

/* one replica's rows of externally supplied draws (NULL: that stream comes from Philox), and where to report how many
 * draws of each stream the replica asked for (the cursors' final values; NULL: not reported) */
typedef struct { const double *targets; uint64_t n_targets; const double *service; uint64_t n_service;
                 uint64_t *arr_used, *svc_used; } otrace;

/* Simulation.__init__ of one replica: entity state, output cursors, the sources' first ticks */
static void orun_init(orun *Rp, const hs_model_desc *m, const hs_run_params *p, uint32_t r,
                      const hs_outputs *out, const otrace *tr)
{
#define R (*Rp)
    memset(&R, 0, sizeof R);
#ifdef HS_ORACLE_HIGH_WATER
    R.heap.clock = INT64_MIN;
#endif
    R.m = m; R.p = p; R.r = r; R.out = out;
    if (tr) { R.trace_targets = tr->targets; R.n_trace_targets = tr->n_targets;
              R.trace_service = tr->service; R.n_trace_service = tr->n_service; }
    uint32_t ne = m->n_entities;
    uint32_t gidx = p->replica_index_base + r;
    uint32_t cell = p->replicas_per_cell ? gidx / p->replicas_per_cell : 0;
    if (m->n_cells) cell %= m->n_cells;
    R.seed = p->seed + (uint64_t)gidx * p->seed_stride;
    R.rid = p->rid_base + gidx * p->rid_stride;
    R.ents = (oent *)calloc(ne, sizeof(oent));
    for (uint32_t i = 0; i < ne; ++i) {
        oent *E = &R.ents[i];
        E->d = m->entities[i];
        if (m->n_cells && m->cell_d0) E->d.d0 = m->cell_d0[(size_t)cell * ne + i];
        if (m->n_cells && m->cell_i0) E->d.i0 = m->cell_i0[(size_t)cell * ne + i];
        E->mn = INFINITY; E->mx = -INFINITY;
        if (E->d.kind == HS_ENT_SERVER && E->d.i2 == HS_SVC_EXPONENTIAL) E->lambda = 1.0 / E->d.d0;
    }
    {   /* SKETCH rows: state lives in the caller's buffer (zeroed here), hs_sketch_layout */
        uint64_t total = 0;
        uint64_t *off = (uint64_t *)calloc(ne, sizeof(uint64_t));
        hs_sketch_layout_impl(m, off, NULL, &total, NULL);
        if (out->sketches && total) {
            uint8_t *base = out->sketches + (size_t)r * total;
            memset(base, 0, total);
            for (uint32_t i = 0; i < ne; ++i) {
                if (R.ents[i].d.kind == HS_ENT_SKETCH) R.ents[i].sk_state = base + off[i];
                if (R.ents[i].d.kind == HS_ENT_CACHE_SERVER) R.ents[i].cache_ins = (double *)(base + off[i]);
            }
        }
        for (uint32_t i = 0; i < ne; ++i)     /* the cache is state the run needs, with or without an output buffer */
            if (R.ents[i].d.kind == HS_ENT_CACHE_SERVER && !R.ents[i].cache_ins) {
                R.ents[i].cache_ins = (double *)calloc((size_t)R.ents[i].d.i0 + 1, sizeof(double));
                R.ents[i].cache_own = 1;
            }
        free(off);
    }
    if (out->records) R.rec = out->records + (size_t)r * p->record_cap;
    if (out->sink_samples) R.smp = out->sink_samples + (size_t)r * p->sample_cap;
    if (out->service_samples) R.svc = out->service_samples + (size_t)r * p->service_cap;
    if (out->histograms && (p->flags & HS_RUN_HISTOGRAM)) {
        R.hist = out->histograms + (size_t)r * HS_HISTOGRAM_BINS;
        memset(R.hist, 0, HS_HISTOGRAM_BINS * sizeof(uint32_t));
    }

    /* Simulation.__init__: reset_event_counter(); source.start() for each source
     * in order; the SourceEvent takes its index from the GLOBAL counter
     * (simulation.py:77,145-154; source.py:120-140). */
    R.counter = 0;
    R.now = 0;
    for (uint32_t i = 0; i < ne; ++i) {
        oent *E = &R.ents[i];
        if (E->d.kind != HS_ENT_SOURCE) continue;
        E->cur_ns = 0;                    /* provider.current_time = start_time   */
        int64_t first = next_arrival(&R, (int)i, E);
        if (first == HS_T_EXHAUSTED) continue;   /* source.start(): RuntimeError -> no tick, source.py:138-140 */
        oev tick = new_event(&R, first, HS_EV_SOURCE_TICK, (int)i);
        heap_push(&R.heap, &tick);
    }
    /* run(): _active_sim_context installs the per-heap counter, again from 0
     * (event_heap.py:48, sim_future.py:64-73). */
    R.counter = 0;
    R.processed = 0;
    R.hash = HS_HASH_INIT;
#undef R
}

/* _execute_until(end_ns) (simulation.py:449-505): the test is on the LAST processed time, so the first event
 * beyond end_ns is still processed.  cut_ns >= 0: stop before the first event later than cut_ns instead (a run cut
 * at an event boundary, hs_run_params.window_end_ns). */
static void orun_until(orun *Rp, int64_t end_ns, int64_t cut_ns)
{
#define R (*Rp)
    const hs_run_params *p = R.p;
    while (R.heap.n && R.now <= end_ns) {
        /* the limit before the cut: a replica that has processed max_events has stopped (hs_run_params.max_events),
         * whether or not its next event lies beyond the window -- as every engine decides it */
        if (p->max_events > 0 && R.processed >= p->max_events) { R.status |= HS_ST_EVENT_LIMIT; break; }
        if (cut_ns >= 0 && R.heap.a[0].time > cut_ns) break;
        oev e = heap_pop(&R.heap);
#ifdef HS_ORACLE_HIGH_WATER
        if (e.hw_future) { R.heap.n_future--; HS_HW_MAX(R.heap.hw[HS_HW_NOW_POP], R.heap.n_now); }
        else R.heap.n_now--;
#endif
        if (e.time < R.now) continue;     /* "time travel": skipped, not counted (simulation.py:479-489) */
        R.now = e.time;
#ifdef HS_ORACLE_HIGH_WATER
        R.heap.clock = R.now;
#endif
        uint64_t w1 = hs_record_word1(e.idx, (uint32_t)e.kind, (uint32_t)e.ent);
        R.hash = hs_hash_step(R.hash, e.time, w1);
        if (R.rec && p->record_cap) {
            hs_event_record *rc = &R.rec[R.processed % (int64_t)p->record_cap];
            rc->time_ns = e.time; rc->sort_index = (uint32_t)e.idx;
            rc->kind = (uint8_t)e.kind; rc->pad = 0; rc->entity = (uint16_t)e.ent;
        }
        if (!(p->flags & HS_RUN_ORDER_HASH)) R.hash = 0;
        R.processed++;
        handle(&R, &e);
    }
#ifdef HS_ORACLE_HIGH_WATER
    R.heap.clock = INT64_MIN;             /* what a barrier delivers next is scheduled from outside the run */
#endif
#undef R
}

static void orun_finish(orun *Rp)
{
#define R (*Rp)
    const hs_outputs *out = R.out; const uint32_t r = R.r; const uint32_t ne = R.m->n_entities;
    /* with the hash off the summary holds 0, as on every engine -- also for a replica that has processed no event */
    const int64_t processed = R.processed; const uint64_t h = (R.p->flags & HS_RUN_ORDER_HASH) ? R.hash : 0;
    if (out->summaries) {
        hs_replica_summary *s = &out->summaries[r];
        s->events_processed = processed; s->final_time_ns = R.now; s->order_hash = h;
        s->next_sort_index = R.counter; s->n_sink_samples = R.n_smp; s->n_service_samples = R.n_svc; s->heap_left = (int32_t)R.heap.n; s->status = R.status;
    }
    if (out->entity_stats) {
        for (uint32_t i = 0; i < ne; ++i) {
            hs_entity_stats *st = &out->entity_stats[(size_t)r * ne + i];
            oent *E = &R.ents[i];
            memset(st, 0, sizeof *st);
            switch (E->d.kind) {
            case HS_ENT_SOURCE: st->c0 = E->generated_count; st->c1 = E->provider_count; break;
            case HS_ENT_SERVER:
                st->c0 = E->accepted; st->c1 = E->dropped; st->c2 = E->completed; st->c3 = E->rejected;
                st->f0 = E->total_service; break;
            case HS_ENT_SINK:
                st->c0 = E->received; st->f0 = hs_neumaier_result(E->sum, E->comp); st->f1 = E->sumsq; st->f2 = E->mn; st->f3 = E->mx; break;
            case HS_ENT_COUNTER: case HS_ENT_REMOTE: st->c0 = E->received; break;
            case HS_ENT_PROBE:
                st->c0 = E->received; st->f0 = hs_neumaier_result(E->sum, E->comp); st->f2 = E->mn; st->f3 = E->mx; break;
            case HS_ENT_SKETCH: st->c0 = E->sk_processed; st->c1 = E->sk_added; break;
            case HS_ENT_CACHE_SERVER:
                st->c0 = E->accepted; st->c1 = E->dropped; st->c2 = E->completed; st->c3 = E->cache_misses;
                st->f0 = (double)E->cache_hits; st->f1 = (double)E->cache_size; break;
            case HS_ENT_LB:
                st->c0 = E->lb_received; st->c1 = E->lb_forwarded; st->c2 = E->lb_in_flight; st->c3 = E->lb_responses; break;
            }
        }
    }
    for (uint32_t i = 0; i < ne; ++i) { free(R.ents[i].q); if (R.ents[i].cache_own) free(R.ents[i].cache_ins); }
    free(R.ents); free(R.heap.a);
#undef R
}

#ifdef HS_ORACLE_HIGH_WATER
/* where run_replica / hs_oracle_run_linked write the rows (set by the *_high_water entry points; one per thread, so
 * slices of an ensemble can run on a thread pool) */
static _Thread_local uint32_t *hw_rows;
static _Thread_local uint32_t *const *hw_part_rows;

static void hw_publish(const orun *R, uint32_t *row)
{
    memcpy(row, R->heap.hw, sizeof R->heap.hw);
    for (uint32_t i = 0; i < R->m->n_entities; ++i) row[HS_HW_FIELDS + i] = R->ents[i].hw_queue;
}
#endif

static void run_replica(const hs_model_desc *m, const hs_run_params *p, uint32_t r,
                        const hs_outputs *out, const otrace *tr)
{
    orun R;
    orun_init(&R, m, p, r, out, tr);
    /* windowed run (core/simulation.py:527-541 cut at event boundaries): pause before the first event later
     * than the window end; resume is not modelled here -- a paused prefix is compared against the device's. */
    const int windowed = (p->window_end_ns >= 0 && p->window_end_ns < p->end_ns);
    orun_until(&R, p->end_ns, windowed ? p->window_end_ns : -1);
    if (tr && tr->arr_used) *tr->arr_used = R.np_cursor;
    if (tr && tr->svc_used) *tr->svc_used = R.py_cursor;
#ifdef HS_ORACLE_HIGH_WATER
    if (hw_rows) hw_publish(&R, hw_rows + (size_t)r * (HS_HW_FIELDS + m->n_entities));
#endif
    orun_finish(&R);
}

/* ---- exported --------------------------------------------------------- */

int hs_oracle_run(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out)
{
    if (!m || !p || !out || m->abi_version != HS_ABI_VERSION) return HS_ERR_INVALID;
    for (uint32_t r = 0; r < p->n_replicas; ++r) run_replica(m, p, r, out, NULL);
    return HS_OK;
}

/* ---- linked partitions: ParallelSimulation with PartitionLinks (parallel/simulation.py:31-284) ------------
 * One orun per partition; WindowedCoordinator.run (coordinator.py:75-172): for every window, every partition runs
 * _run_window(window_end) = _execute_until(window_end) -- the per-heap sort-index counters make the partitions'
 * results independent of the order the thread pool runs them in (event_heap.py:46-48) -- then _exchange_events
 * (coordinator.py:182-227) walks the outboxes in partition order: one loss draw from the coordinator's generator
 * when the link loses packets, event.time = send_time + link.latency.sample(), Simulation.schedule() = heap push.
 * links[p][k] / link_dst[p][k]: the link a REMOTE row with i0 = k of partition p sends through, and the partition
 * it ends in.  window_ends: the coordinator's window ends in ns (computed in float seconds by the host layer,
 * coordinator.py:88-95).  The coordinator's draws: HS_STREAM_LINK_LOSS / HS_STREAM_LINK_LATENCY | stream << 8 of
 * Philox key cseed + g * cseed_stride, replica word crid_base + g * crid_stride (g = global replica index). */
int hs_oracle_run_linked(uint32_t n_parts, const hs_model_desc *const *models, const hs_run_params *const *params,
                         const hs_outputs *const *outs, const hs_link_desc *const *links, const uint32_t *const *link_dst,
                         const int64_t *window_ends, uint32_t n_windows, uint32_t n_streams,
                         uint64_t cseed, uint64_t cseed_stride, uint32_t crid_base, uint32_t crid_stride,
                         uint64_t *delivered, uint64_t *lost)
{
    if (!n_parts || !models || !params || !outs || !window_ends) return HS_ERR_INVALID;
    for (uint32_t q = 0; q < n_parts; ++q)
        if (!models[q] || models[q]->abi_version != HS_ABI_VERSION || params[q]->n_replicas != params[0]->n_replicas) return HS_ERR_INVALID;
    const uint32_t n = params[0]->n_replicas;
    orun *R = (orun *)calloc(n_parts, sizeof(orun));
    uint64_t *lat_draws = (uint64_t *)calloc(n_streams ? n_streams : 1, sizeof(uint64_t));
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t g = params[0]->replica_index_base + r;
        const uint64_t seed = cseed + (uint64_t)g * cseed_stride;
        const uint32_t rid = crid_base + g * crid_stride;
        uint64_t loss_draws = 0, n_del = 0, n_lost = 0;
        memset(lat_draws, 0, (n_streams ? n_streams : 1) * sizeof(uint64_t));
        for (uint32_t q = 0; q < n_parts; ++q) {
            orun_init(&R[q], models[q], params[q], r, outs[q], NULL);
            R[q].outbox_cap = models[q]->outbox_cap;
            R[q].outbox = (hs_xevent *)calloc(R[q].outbox_cap ? R[q].outbox_cap : 1, sizeof(hs_xevent));
        }
        for (uint32_t w = 0; w < n_windows; ++w) {
            for (uint32_t q = 0; q < n_parts; ++q) orun_until(&R[q], window_ends[w], -1);      /* 1. EXECUTE */
#ifdef HS_ORACLE_HIGH_WATER
            for (uint32_t q = 0; q < n_parts; ++q) R[q].hw_received = 0;
#endif
            for (uint32_t q = 0; q < n_parts; ++q) {                                            /* 2. EXCHANGE */
                for (uint32_t k = 0; k < R[q].outbox_n; ++k) {
                    const hs_xevent *x = &R[q].outbox[k];
                    const hs_entity_desc *rem = &models[q]->entities[x->ent];
                    const hs_link_desc *lk = &links[q][rem->i0];
                    orun *D = &R[link_dst[q][rem->i0]];
                    if (lk->packet_loss > 0.0 &&
                        hs_uniform(seed, rid, HS_STREAM_LINK_LOSS, loss_draws++) < lk->packet_loss) { n_lost++; continue; }
                    int64_t lat;
                    if (lk->latency_kind == HS_SVC_EXPONENTIAL) {
                        const double u = hs_uniform(seed, rid, HS_STREAM_LINK_LATENCY | ((uint32_t)lk->stream << 8), lat_draws[lk->stream]++);
                        lat = hs_exp_latency_ns(u, 1.0 / lk->latency_mean_s);
                    } else lat = hs_seconds_to_ns(lk->latency_mean_s);
                    oev e; memset(&e, 0, sizeof e);
                    e.time = x->time_ns + lat; e.idx = x->sort_index; e.ent = rem->i1;
                    e.kind = request_kind_for(D, rem->i1);
                    e.created_at = x->created_ns; e.key = x->key; e.lb_hook = -1; e.poll_hook = -1;
                    heap_push(&D->heap, &e);
                    n_del++;
#ifdef HS_ORACLE_HIGH_WATER
                    D->hw_received++; HS_HW_MAX(D->heap.hw[HS_HW_INBOX], D->hw_received);
#endif
                }
                R[q].outbox_n = 0;
#ifdef HS_ORACLE_HIGH_WATER
                R[q].hw_sent = 0;
#endif
            }
        }
#ifdef HS_ORACLE_HIGH_WATER
        if (hw_part_rows)
            for (uint32_t q = 0; q < n_parts; ++q) hw_publish(&R[q], hw_part_rows[q] + (size_t)r * (HS_HW_FIELDS + models[q]->n_entities));
#endif
        for (uint32_t q = 0; q < n_parts; ++q) { free(R[q].outbox); orun_finish(&R[q]); }
        if (delivered) delivered[r] = n_del;
        if (lost) lost[r] = n_lost;
    }
    free(lat_draws); free(R);
    return HS_OK;
}

/* Run replicas [r0, r1) only: lets Python spread a batch over host processes/threads. */
int hs_oracle_run_range(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out,
                        uint32_t r0, uint32_t r1)
{
    if (!m || !p || !out || m->abi_version != HS_ABI_VERSION) return HS_ERR_INVALID;
    for (uint32_t r = r0; r < r1 && r < p->n_replicas; ++r) run_replica(m, p, r, out, NULL);
    return HS_OK;
}

#ifdef HS_ORACLE_HIGH_WATER
/* hs_oracle_run_range that also fills hw[n_replicas][HS_HW_FIELDS + n_entities] (rows [r0, r1) only) */
int hs_oracle_high_water_range(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out,
                               uint32_t r0, uint32_t r1, uint32_t *hw)
{
    hw_rows = hw;
    const int rc = hs_oracle_run_range(m, p, out, r0, r1);
    hw_rows = NULL;
    return rc;
}

/* hs_oracle_run_linked that also fills hw[q][n_replicas][HS_HW_FIELDS + n_entities of partition q] */
int hs_oracle_high_water_linked(uint32_t n_parts, const hs_model_desc *const *models, const hs_run_params *const *params,
                                const hs_outputs *const *outs, const hs_link_desc *const *links, const uint32_t *const *link_dst,
                                const int64_t *window_ends, uint32_t n_windows, uint32_t n_streams,
                                uint64_t cseed, uint64_t cseed_stride, uint32_t crid_base, uint32_t crid_stride,
                                uint64_t *delivered, uint64_t *lost, uint32_t *const *hw)
{
    hw_part_rows = hw;
    const int rc = hs_oracle_run_linked(n_parts, models, params, outs, links, link_dst, window_ends, n_windows, n_streams,
                                        cseed, cseed_stride, crid_base, crid_stride, delivered, lost);
    hw_part_rows = NULL;
    return rc;
}
#endif

/* CPU anchor for bench.py: n_threads POSIX threads pull replica indices [0, max_replicas) from a shared
 * counter and run them until budget_s of wall time is spent (a replica in progress is finished), all inside
 * C -- no Python call, GIL hand-over or ctypes marshalling per replica.  Every thread keeps private totals;
 * only the summary of the replica it runs is written (into a thread-local hs_replica_summary).
 * Returns events processed / replicas completed / wall seconds. */
#include <pthread.h>
#include <stdatomic.h>
#include <time.h>
typedef struct { const hs_model_desc *m; const hs_run_params *p; atomic_uint *next; uint32_t max_replicas;
                 double deadline; int64_t events; uint32_t replicas; } obench_arg;
static double obench_now(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec; }
static void *obench_worker(void *v)
{
    obench_arg *a = (obench_arg *)v;
    hs_run_params q = *a->p;
    q.n_replicas = 1; q.record_cap = q.sample_cap = q.service_cap = 0;
    const uint32_t ne = a->m->n_entities;
    hs_replica_summary summ; hs_entity_stats *st = (hs_entity_stats *)calloc(ne ? ne : 1, sizeof *st);
    hs_outputs o; memset(&o, 0, sizeof o); o.summaries = &summ; o.entity_stats = st;
    while (obench_now() < a->deadline) {
        const uint32_t k = atomic_fetch_add(a->next, 1u);
        if (k >= a->max_replicas) break;
        q.replica_index_base = a->p->replica_index_base + k;     /* global replica id k: its own Philox streams */
        memset(&summ, 0, sizeof summ);
        run_replica(a->m, &q, 0, &o, NULL);
        a->events += summ.events_processed; a->replicas += 1;
    }
    free(st);
    return NULL;
}
int hs_oracle_bench(const hs_model_desc *m, const hs_run_params *p, int n_threads, double budget_s, uint32_t max_replicas,
                    int64_t *events, uint32_t *replicas, double *wall_s)
{
    if (!m || !p || m->abi_version != HS_ABI_VERSION || n_threads < 1 || n_threads > 4096) return HS_ERR_INVALID;
    atomic_uint next = 0;
    pthread_t *th = (pthread_t *)calloc((size_t)n_threads, sizeof *th);
    obench_arg *args = (obench_arg *)calloc((size_t)n_threads, sizeof *args);
    const double t0 = obench_now();
    for (int i = 0; i < n_threads; ++i) {
        args[i].m = m; args[i].p = p; args[i].next = &next; args[i].max_replicas = max_replicas; args[i].deadline = t0 + budget_s;
        pthread_create(&th[i], NULL, obench_worker, &args[i]);
    }
    int64_t ev = 0; uint32_t rp = 0;
    for (int i = 0; i < n_threads; ++i) { pthread_join(th[i], NULL); ev += args[i].events; rp += args[i].replicas; }
    if (events) *events = ev;
    if (replicas) *replicas = rp;
    if (wall_s) *wall_s = obench_now() - t0;
    free(th); free(args);
    return HS_OK;
}

/* Replicas driven by externally supplied draws: arrival target areas (-log(1-U), poisson_arrival.py:31) and
 * service samples (random.expovariate, exponential.py:43) captured from the reference's stock generators.  The
 * draws are laid out as hs_set_trace lays them out, one row per replica slot: targets[n_replicas][n_targets],
 * service[n_replicas][n_service]; a stream with no draws (NULL or n = 0) comes from Philox, as on the device.  The
 * cell of a replica follows replica_index_base and replicas_per_cell, as in hs_oracle_run.  A replica that asks for
 * a draw past the end of its row gets a target of 1e300 (no further arrival, an unbounded service time) and runs on;
 * arr_used / svc_used (per replica slot, each optional) receive how many draws of each stream the replica asked
 * for, so a caller learns what every replica needed.  Replicas [r0, r1) only, so Python can spread a batch over
 * threads (r1 is clamped to n_replicas). */
int hs_oracle_run_trace_range(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out,
                              const double *targets, uint64_t n_targets, const double *service, uint64_t n_service,
                              uint32_t r0, uint32_t r1, uint64_t *arr_used, uint64_t *svc_used)
{
    if (!m || !p || !out || m->abi_version != HS_ABI_VERSION) return HS_ERR_INVALID;
    if (!targets) n_targets = 0;
    if (!service) n_service = 0;
    for (uint32_t r = r0; r < r1 && r < p->n_replicas; ++r) {
        otrace tr = { n_targets ? targets + (size_t)r * n_targets : NULL, n_targets,
                      n_service ? service + (size_t)r * n_service : NULL, n_service,
                      arr_used ? arr_used + r : NULL, svc_used ? svc_used + r : NULL };
        run_replica(m, p, r, out, &tr);
    }
    return HS_OK;
}

/* Every replica of hs_oracle_run_trace_range, without the draw counts. */
int hs_oracle_run_trace(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out,
                        const double *targets, uint64_t n_targets, const double *service, uint64_t n_service)
{
    if (!p) return HS_ERR_INVALID;
    return hs_oracle_run_trace_range(m, p, out, targets, n_targets, service, n_service, 0, p->n_replicas, NULL, NULL);
}

int hs_sketch_layout(const hs_model_desc *m, uint64_t *per_replica, uint64_t *merged, uint64_t *total, uint64_t *merged_total)
{
    if (!m || !m->entities) return HS_ERR_INVALID;
    hs_sketch_layout_impl(m, per_replica, merged, total, merged_total);
    return HS_OK;
}

/* CPU twins of the shared sampler, called by the Philox plug-ins that
 * tests/golden/gen_golden.py injects into the unmodified reference. */
double hs_cpu_uniform(uint64_t seed, uint32_t replica, uint32_t sid, uint64_t draw)
{ return hs_uniform(seed, replica, sid, draw); }
double hs_cpu_log(double x) { return hs_log(x); }
double hs_cpu_exp1(double u) { return hs_exp1(u); }
int64_t hs_cpu_seconds_to_ns(double s) { return hs_seconds_to_ns(s); }
double hs_cpu_ns_to_seconds(int64_t ns) { return hs_ns_to_seconds(ns); }
int64_t hs_cpu_next_arrival_ns(int64_t cur, double target, double rate) { return hs_next_arrival_ns(cur, target, rate); }
int64_t hs_cpu_exp_latency_ns(double u, double lambda) { return hs_exp_latency_ns(u, lambda); }
uint32_t hs_cpu_latency_bin(int64_t lat_ns) { return hs_latency_bin(lat_ns); }
uint64_t hs_cpu_hash_step(uint64_t h, int64_t t, uint64_t idx, uint32_t kind, uint32_t ent)
{ return hs_hash_step(h, t, hs_record_word1(idx, kind, ent)); }
int64_t hs_cpu_next_arrival_profile_ns(int32_t kind, double p0, double p1, double p2, double p3, int64_t cur, double target)
{ hs_profile_desc P; P.kind = kind; P.pad = 0; P.p[0] = p0; P.p[1] = p1; P.p[2] = p2; P.p[3] = p3;
  return hs_next_arrival_profile_ns(&P, cur, target); }
double hs_cpu_integrate_rate(int32_t kind, double p0, double p1, double p2, double p3, double a, double b)
{ hs_profile_desc P; P.kind = kind; P.pad = 0; P.p[0] = p0; P.p[1] = p1; P.p[2] = p2; P.p[3] = p3;
  return hs_integrate_rate(&P, a, b); }
/* the shared sketch steps of csrc/hs_sketch.h, callable on their own (tests/test_sketch_kats.py feeds them the
 * streams whose answers the reference's sketch classes gave) */
void hs_cpu_sketch_add(uint8_t *state, const int32_t *tab, int32_t algo, int32_t p_or_depth, int32_t width, int64_t K, int32_t key)
{ hs_sketch_add(state, tab, algo, p_or_depth, width, K, key); }
void hs_cpu_hll_hash(uint64_t seed, int32_t p, int32_t key, int32_t *idx, int32_t *run) { hs_hll_hash(seed, p, key, idx, run); }
uint64_t hs_cpu_cms_row_seed(uint64_t seed, int32_t row) { return hs_cms_row_seed(seed, row); }
int32_t hs_cpu_cms_col(uint64_t row_seed, int32_t width, int32_t key) { return hs_cms_col(row_seed, width, key); }
int32_t hs_cpu_bloom_bit(uint64_t seed, int32_t i, int32_t size_bits, int32_t key) { return hs_bloom_bit(seed, i, size_bits, key); }
int hs_cpu_tdigest_add(uint8_t *state, double compression, uint32_t buf_size, uint32_t cap, double value)
{ return hs_tdigest_add(state, compression, buf_size, cap, value); }
int32_t hs_cpu_routing_key(double u, int32_t n, const double *cum_probs) { return hs_routing_key(u, n, cum_probs); }
void hs_cpu_philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t *out4)
{ hs_u32x4 r = hs_philox4x32_10(c0, c1, c2, c3, k0, k1); out4[0] = r.x; out4[1] = r.y; out4[2] = r.z; out4[3] = r.w; }
