/* priority_oracle.c -- the CPU oracle (oracle/hs_oracle.c) with PriorityQueue servers.  TEST INFRASTRUCTURE ONLY.
 *
 * A server whose row has i1 = HS_Q_PRIORITY keeps its queue in the oracle's unchanged deque, in insertion order.
 * PriorityQueue.pop (components/queue_policy.py:263-267) returns the entry with the smallest (priority, insert_order)
 * (queue_policy.py:197-210, a total order): in a deque kept in insertion order that is the FIRST entry whose priority
 * is the smallest.  Before a POLL at such a server, po_front moves that entry to the front of the deque, the others
 * keeping their order, and the oracle's own handler pops the front as it pops a FIFOQueue.  The priority of an entry
 * is table[routing key], the server's table in profile_table at i3 - 1 (include/hs_b200.h).  This is a linear scan,
 * not a heap: the device's binary heap is checked against a different algorithm.  Everything else -- push, drop,
 * NOTIFY, the Probe's depth (len(heap) = the deque's length) -- is the oracle's FIFO code, as the reference's Queue
 * protocol around the policy is the same for every policy.
 * Built by tests/priority_oracle_lib.py into a temporary directory. */
#include "../oracle/hs_oracle.c"

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

/* orun_until with po_front before every handler */
static void po_until(orun *Rp, int64_t end_ns, int64_t cut_ns)
{
#define R (*Rp)
    const hs_run_params *p = R.p;
    while (R.heap.n && R.now <= end_ns) {
        if (p->max_events > 0 && R.processed >= p->max_events) { R.status |= HS_ST_EVENT_LIMIT; break; }
        if (cut_ns >= 0 && R.heap.a[0].time > cut_ns) break;
        oev e = heap_pop(&R.heap);
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
        po_front(&R, &e);
        handle(&R, &e);
    }
#undef R
}

int hs_priority_oracle_run_range(const hs_model_desc *m, const hs_run_params *p, const hs_outputs *out, uint32_t r0, uint32_t r1)
{
    if (!m || !p || !out || m->abi_version != HS_ABI_VERSION) return HS_ERR_INVALID;
    for (uint32_t r = r0; r < r1 && r < p->n_replicas; ++r) {
        orun R;
        orun_init(&R, m, p, r, out, NULL);
        const int windowed = (p->window_end_ns >= 0 && p->window_end_ns < p->end_ns);
        po_until(&R, p->end_ns, windowed ? p->window_end_ns : -1);
        orun_finish(&R);
    }
    return HS_OK;
}

/* hs_oracle_run_linked (oracle/hs_oracle.c) with po_until running each partition's window; the exchange step is the
 * oracle's, restated here */
int hs_priority_oracle_run_linked(uint32_t n_parts, const hs_model_desc *const *models, const hs_run_params *const *params,
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
            for (uint32_t q = 0; q < n_parts; ++q) po_until(&R[q], window_ends[w], -1);          /* 1. EXECUTE */
            for (uint32_t q = 0; q < n_parts; ++q) {                                              /* 2. EXCHANGE */
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
                }
                R[q].outbox_n = 0;
            }
        }
        for (uint32_t q = 0; q < n_parts; ++q) { free(R[q].outbox); orun_finish(&R[q]); }
        if (delivered) delivered[r] = n_del;
        if (lost) lost[r] = n_lost;
    }
    free(lat_draws); free(R);
    return HS_OK;
}
