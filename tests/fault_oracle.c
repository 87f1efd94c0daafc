/* fault_oracle.c -- the CPU oracle (oracle/hs_oracle.c) with node faults.  TEST INFRASTRUCTURE ONLY.
 *
 * The oracle restates Simulation.run() one to one; this file adds, around its unchanged heap, handlers and
 * bookkeeping, what faults change in the reference (paths under happysimulator/):
 *   bootstrap   core/simulation.py:162-169  FaultSchedule.start() after the sources and probes: one Event.once per
 *                                           HS_ENT_FAULT row, sort index = the row's i3 (global counter)
 *   the loop    core/simulation.py:470-505  a cancelled event is popped, counted (events_cancelled) and skipped before
 *                                           anything else -- it is not processed and does not move the clock
 *   the drop    core/event.py:261-262       Event.invoke of an event whose target has _crashed set returns []: the event
 *                                           counts and is recorded, neither its handler nor its completion hooks run.
 *                                           The targets a request-kind event names are the entity itself; NOTIFY, POLL,
 *                                           DELIVER, WORKER and CONTINUATION target the hidden queue / driver / worker,
 *                                           which no fault can name
 *   the flag    faults/node_faults.py:41-128  a boolean: the last FAULT event processed decides
 * heapq is restated move for move, so ties of an in-run event with a pending FAULT event are ordered as the reference
 * orders them; HS_ST_FAULT_TIE is set when such a tie occurs, as the engines set it.
 * Built by tests/fault_oracle_lib.py into a temporary directory. */
#include "../oracle/hs_oracle.c"

#define FO_DROPPABLE ((1u << HS_EV_SOURCE_TICK) | (1u << HS_EV_REQ_LB) | (1u << HS_EV_REQ_ENQUEUE) | (1u << HS_EV_REQ_SINK) | \
                      (1u << HS_EV_LB_RESPONSE) | (1u << HS_EV_REQ_COUNTER) | (1u << HS_EV_REQ_SKETCH))

typedef struct { uint8_t *crashed; int64_t *fired, *cancelled; uint32_t f0, ne; } ofault;

/* a FAULT row that has neither fired nor been popped cancelled */
static int fo_pending(const ofault *F, uint32_t i) { return F->fired[i] == 0 && F->cancelled[i] == 0; }

/* an event created by the last handler (sort index in [c0, c1), or the WORKER a DELIVER re-pushes with its payload's
 * index) with the key of a pending FAULT event: HS_ST_FAULT_TIE */
static void fo_tie(orun *R, const ofault *F, uint64_t c0, uint64_t c1, int have_payload, uint64_t payload_idx)
{
    for (uint32_t i = F->f0; i < F->ne; ++i) {
        if (!fo_pending(F, i)) continue;
        const uint64_t fi = (uint64_t)(uint32_t)R->m->entities[i].i3;
        const int64_t ft = R->m->entities[i].l0;
        if (!((fi >= c0 && fi < c1) || (have_payload && fi == payload_idx))) continue;
        for (size_t k = 0; k < R->heap.n; ++k) {
            const oev *e = &R->heap.a[k];
            if (e->time == ft && e->idx == fi && !(e->kind == HS_EV_FAULT && (uint32_t)e->ent == i)) { R->status |= HS_ST_FAULT_TIE; return; }
        }
    }
}

static void fo_until(orun *Rp, ofault *F, int64_t end_ns, int64_t cut_ns)
{
#define R (*Rp)
    const hs_run_params *p = R.p;
    while (R.heap.n && R.now <= end_ns) {
        if (p->max_events > 0 && R.processed >= p->max_events) { R.status |= HS_ST_EVENT_LIMIT; break; }
        if (cut_ns >= 0 && R.heap.a[0].time > cut_ns) break;
        oev e = heap_pop(&R.heap);
        if (e.kind == HS_EV_FAULT && R.ents[e.ent].d.i2) { F->cancelled[e.ent]++; continue; }   /* event._cancelled */
        if (e.time < R.now) continue;
        R.now = e.time;
        uint64_t w1 = hs_record_word1(e.idx, (uint32_t)e.kind, (uint32_t)e.ent);
        R.hash = hs_hash_step(R.hash, e.time, w1);
        if (R.rec && p->record_cap) {
            hs_event_record *rc = &R.rec[R.processed % (int64_t)p->record_cap];
            rc->time_ns = e.time; rc->sort_index = (uint32_t)e.idx;
            rc->kind = (uint8_t)e.kind; rc->pad = 0; rc->entity = (uint16_t)e.ent;
        }
        if (!(p->flags & HS_RUN_ORDER_HASH)) R.hash = 0;
        R.processed++;
        if (e.kind == HS_EV_FAULT) {                          /* the CallbackEntity's fn: entity._crashed = True / False */
            F->crashed[R.ents[e.ent].d.target] = (uint8_t)R.ents[e.ent].d.i1;
            F->fired[e.ent]++;
            continue;
        }
        if (F->crashed[e.ent] && ((FO_DROPPABLE >> e.kind) & 1u)) continue;   /* Event.invoke returns [] */
        const uint64_t c0 = R.counter;
        handle(&R, &e);
        if (F->f0 < F->ne) fo_tie(&R, F, c0, R.counter, e.kind == HS_EV_DELIVER, e.payload_idx);
    }
#undef R
}

static void fo_replica(const hs_model_desc *m, const hs_run_params *p, uint32_t r, const hs_outputs *out)
{
    orun R;
    orun_init(&R, m, p, r, out, NULL);
    ofault F;
    F.ne = m->n_entities; F.f0 = F.ne;
    while (F.f0 > 0 && m->entities[F.f0 - 1].kind == HS_ENT_FAULT) F.f0--;
    F.crashed = (uint8_t *)calloc(F.ne, 1);
    F.fired = (int64_t *)calloc(F.ne, sizeof(int64_t));
    F.cancelled = (int64_t *)calloc(F.ne, sizeof(int64_t));
    for (uint32_t i = F.f0; i < F.ne; ++i) {                  /* FaultSchedule.start(): pushed after the sources */
        oev f; memset(&f, 0, sizeof f);
        f.time = m->entities[i].l0; f.idx = (uint64_t)(uint32_t)m->entities[i].i3; f.kind = HS_EV_FAULT; f.ent = (int32_t)i;
        f.key = -1; f.lb_hook = -1; f.poll_hook = -1;
        heap_push(&R.heap, &f);
    }
    const int windowed = (p->window_end_ns >= 0 && p->window_end_ns < p->end_ns);
    fo_until(&R, &F, p->end_ns, windowed ? p->window_end_ns : -1);
    orun_finish(&R);
    if (out->entity_stats)
        for (uint32_t i = F.f0; i < F.ne; ++i) {
            hs_entity_stats *st = &out->entity_stats[(size_t)r * F.ne + i];
            st->c0 = F.fired[i]; st->c1 = F.cancelled[i];
        }
    free(F.crashed); free(F.fired); free(F.cancelled);
}

int hs_fault_oracle_run_range(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out, uint32_t r0, uint32_t r1)
{
    if (!m || !p || !out || m->abi_version != HS_ABI_VERSION) return HS_ERR_INVALID;
    for (uint32_t r = r0; r < r1 && r < p->n_replicas; ++r) fo_replica(m, p, r, out);
    return HS_OK;
}
