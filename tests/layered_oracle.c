/* layered_oracle.c -- the CPU oracle (oracle/hs_oracle.c, included unchanged) with the layers the tests put around its
 * heap, handlers and bookkeeping: node faults, PriorityQueue servers, and linked runs whose replicas are sweep cells.
 * TEST INFRASTRUCTURE ONLY.  A model with neither FAULT rows nor priority servers runs as orun_until runs it.
 *
 * Node faults, as the reference has them (paths under happysimulator/):
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
 *
 * PriorityQueue servers (a SERVER row with i1 = HS_Q_PRIORITY) keep their queue in the oracle's unchanged deque, in
 * insertion order.  PriorityQueue.pop (components/queue_policy.py:263-267) returns the entry with the smallest
 * (priority, insert_order) (queue_policy.py:197-210, a total order): in a deque kept in insertion order that is the
 * FIRST entry whose priority is the smallest.  Before a POLL at such a server, po_front moves that entry to the front
 * of the deque, the others keeping their order, and the oracle's own handler pops the front as it pops a FIFOQueue.
 * The priority of an entry is table[routing key], the server's table in profile_table at i3 - 1 (include/hs_b200.h).
 * This is a linear scan, not a heap: the device's binary heap is checked against a different algorithm.  Everything
 * else -- push, drop, NOTIFY, the Probe's depth -- is the oracle's FIFO code, as the reference's Queue protocol around
 * the policy is the same for every policy.  POLL is not droppable, so po_front and the crash drop never meet.
 *
 * Built by tests/oracle_lib.build() into a temporary directory. */
#include "../oracle/hs_oracle.c"

#define FO_DROPPABLE ((1u << HS_EV_SOURCE_TICK) | (1u << HS_EV_REQ_LB) | (1u << HS_EV_REQ_ENQUEUE) | (1u << HS_EV_REQ_SINK) | \
                      (1u << HS_EV_LB_RESPONSE) | (1u << HS_EV_REQ_COUNTER) | (1u << HS_EV_REQ_SKETCH))

/* the fault layer of one replica: FAULT rows are [f0, ne), the last rows of the model */
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

/* before a POLL at a priority server: its first entry of smallest priority to the front of the deque */
static void po_front(orun *R, const oev *e)
{
    if (e->kind != HS_EV_POLL) return;
    oent *S = &R->ents[e->ent];
    if (S->d.kind != HS_ENT_SERVER || S->d.i1 != HS_Q_PRIORITY || S->q_len < 2) return;
    const double *tab = R->m->profile_table + (S->d.i3 - 1);
    size_t best = 0;
    for (size_t i = 1; i < S->q_len; ++i)
        if (tab[S->q[(S->q_head + i) % S->q_cap].key] < tab[S->q[(S->q_head + best) % S->q_cap].key]) best = i;
    const oreq top = S->q[(S->q_head + best) % S->q_cap];
    for (size_t i = best; i > 0; --i) S->q[(S->q_head + i) % S->q_cap] = S->q[(S->q_head + i - 1) % S->q_cap];
    S->q[S->q_head] = top;
}

/* Simulation.__init__ of one replica: orun_init, then FaultSchedule.start(), pushed after the sources */
static void lo_init(orun *R, ofault *F, const hs_model_desc *m, const hs_run_params *p, uint32_t r, const hs_outputs *out)
{
    orun_init(R, m, p, r, out, NULL);
    F->ne = m->n_entities; F->f0 = F->ne;
    while (F->f0 > 0 && m->entities[F->f0 - 1].kind == HS_ENT_FAULT) F->f0--;
    F->crashed = (uint8_t *)calloc(F->ne, 1);
    F->fired = (int64_t *)calloc(F->ne, sizeof(int64_t));
    F->cancelled = (int64_t *)calloc(F->ne, sizeof(int64_t));
    for (uint32_t i = F->f0; i < F->ne; ++i) {
        oev f; memset(&f, 0, sizeof f);
        f.time = m->entities[i].l0; f.idx = (uint64_t)(uint32_t)m->entities[i].i3; f.kind = HS_EV_FAULT; f.ent = (int32_t)i;
        f.key = -1; f.lb_hook = -1; f.poll_hook = -1;
        heap_push(&R->heap, &f);
    }
}

/* orun_finish, then each FAULT row's statistics: c0 = fired, c1 = popped cancelled */
static void lo_finish(orun *R, ofault *F)
{
    const hs_outputs *out = R->out; const uint32_t r = R->r;
    orun_finish(R);
    if (out->entity_stats)
        for (uint32_t i = F->f0; i < F->ne; ++i) {
            hs_entity_stats *st = &out->entity_stats[(size_t)r * F->ne + i];
            st->c0 = F->fired[i]; st->c1 = F->cancelled[i];
        }
    free(F->crashed); free(F->fired); free(F->cancelled);
}

/* orun_until with the layers: the cancelled-FAULT skip, FAULT firing, the crash drop, po_front before the handler and
 * the tie check after it */
static void lo_until(orun *Rp, ofault *F, int64_t end_ns, int64_t cut_ns)
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
        po_front(&R, &e);
        handle(&R, &e);
        if (F->f0 < F->ne) fo_tie(&R, F, c0, R.counter, e.kind == HS_EV_DELIVER, e.payload_idx);
    }
#undef R
}

int hs_layered_oracle_run_range(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out, uint32_t r0, uint32_t r1)
{
    if (!m || !p || !out || m->abi_version != HS_ABI_VERSION) return HS_ERR_INVALID;
    const int windowed = (p->window_end_ns >= 0 && p->window_end_ns < p->end_ns);
    for (uint32_t r = r0; r < r1 && r < p->n_replicas; ++r) {
        orun R; ofault F;
        lo_init(&R, &F, m, p, r, out);
        lo_until(&R, &F, p->end_ns, windowed ? p->window_end_ns : -1);
        lo_finish(&R, &F);
    }
    return HS_OK;
}

/* hs_oracle_run_linked (oracle/hs_oracle.c) with lo_until running each partition's window.  Every partition's
 * Simulation bootstraps its own FAULT rows (sort indices from its own counter, parallel/simulation.py:94-104).  The
 * exchange is the coordinator's with cells (hs_coordinator_exchange_cells): replica g sends through the link row
 * links[q][cell * n_links[q] + k] of its cell (g / replicas_per_cell) % n_cells, with one loss draw only when that
 * row's loss is > 0, and draws with key cseed + g * cseed_stride and replica word crid_base + g * crid_stride; with
 * n_cells = 1 it is hs_oracle_run_linked's exchange.  The partitions' model cells (cell_d0 / cell_i0) are applied by
 * orun_init.  A delivered event keeps the sender's sort index: one that ties with a pending FAULT event of the
 * receiver sets HS_ST_FAULT_TIE there, as an in-run push does.  The engines schedule what a barrier delivered when the
 * next window starts, so the deliveries of the last barrier (never popped by anyone) are not tested. */
int hs_layered_oracle_run_linked(uint32_t n_parts, const hs_model_desc *const *models, const hs_run_params *const *params,
                                 const hs_outputs *const *outs, const hs_link_desc *const *links, const uint32_t *const *link_dst,
                                 const uint32_t *n_links, uint32_t n_cells, uint32_t replicas_per_cell,
                                 const int64_t *window_ends, uint32_t n_windows, uint32_t n_streams,
                                 uint64_t cseed, uint64_t cseed_stride, uint32_t crid_base, uint32_t crid_stride,
                                 uint64_t *delivered, uint64_t *lost)
{
    if (!n_parts || !models || !params || !outs || !window_ends || !n_cells || !replicas_per_cell) return HS_ERR_INVALID;
    for (uint32_t q = 0; q < n_parts; ++q)
        if (!models[q] || models[q]->abi_version != HS_ABI_VERSION || params[q]->n_replicas != params[0]->n_replicas) return HS_ERR_INVALID;
    const uint32_t n = params[0]->n_replicas;
    orun *R = (orun *)calloc(n_parts, sizeof(orun));
    ofault *F = (ofault *)calloc(n_parts, sizeof(ofault));
    uint64_t *lat_draws = (uint64_t *)calloc(n_streams ? n_streams : 1, sizeof(uint64_t));
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t g = params[0]->replica_index_base + r;
        const uint64_t seed = cseed + (uint64_t)g * cseed_stride;
        const uint32_t rid = crid_base + g * crid_stride;
        const uint32_t cell = (g / replicas_per_cell) % n_cells;
        uint64_t loss_draws = 0, n_del = 0, n_lost = 0;
        memset(lat_draws, 0, (n_streams ? n_streams : 1) * sizeof(uint64_t));
        for (uint32_t q = 0; q < n_parts; ++q) {
            lo_init(&R[q], &F[q], models[q], params[q], r, outs[q]);
            R[q].outbox_cap = models[q]->outbox_cap;
            R[q].outbox = (hs_xevent *)calloc(R[q].outbox_cap ? R[q].outbox_cap : 1, sizeof(hs_xevent));
        }
        for (uint32_t w = 0; w < n_windows; ++w) {
            for (uint32_t q = 0; q < n_parts; ++q) lo_until(&R[q], &F[q], window_ends[w], -1);     /* 1. EXECUTE */
            for (uint32_t q = 0; q < n_parts; ++q) {                                                 /* 2. EXCHANGE */
                for (uint32_t k = 0; k < R[q].outbox_n; ++k) {
                    const hs_xevent *x = &R[q].outbox[k];
                    const hs_entity_desc *rem = &models[q]->entities[x->ent];
                    const hs_link_desc *lk = &links[q][(size_t)cell * n_links[q] + rem->i0];
                    const uint32_t d = link_dst[q][rem->i0];
                    orun *D = &R[d];
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
                    if (w + 1 < n_windows)
                        for (uint32_t i = F[d].f0; i < F[d].ne; ++i)
                            if (fo_pending(&F[d], i) && models[d]->entities[i].l0 == e.time &&
                                (uint64_t)(uint32_t)models[d]->entities[i].i3 == e.idx) D->status |= HS_ST_FAULT_TIE;
                    heap_push(&D->heap, &e);
                    n_del++;
                }
                R[q].outbox_n = 0;
            }
        }
        for (uint32_t q = 0; q < n_parts; ++q) { free(R[q].outbox); lo_finish(&R[q], &F[q]); }
        if (delivered) delivered[r] = n_del;
        if (lost) lost[r] = n_lost;
    }
    free(lat_draws); free(F); free(R);
    return HS_OK;
}
