/* linked_fault_oracle.c -- the fault oracle (tests/fault_oracle.c) for the partitions of a linked ParallelSimulation,
 * each with its own node-fault schedule.  TEST INFRASTRUCTURE ONLY.
 *
 * hs_fault_oracle_run_linked is hs_oracle_run_linked (oracle/hs_oracle.c) with fo_until running each partition's
 * window: every partition's Simulation bootstraps its own FAULT rows (sort indices from its own counter,
 * parallel/simulation.py:94-104), and the exchange step is the oracle's, restated here.  A delivered event keeps the
 * sender's sort index: one that ties with a pending FAULT event of the receiver sets HS_ST_FAULT_TIE there, as an
 * in-run push does.  The engines schedule what a barrier delivered when the next window starts, so the deliveries of
 * the last barrier (never popped by anyone) are not tested.
 * Built by tests/linked_fault_oracle_lib.py into a temporary directory. */
#include "fault_oracle.c"

/* Simulation.__init__ of one partition's replica: orun_init, then FaultSchedule.start() (fo_replica's bootstrap) */
static void lfo_init(orun *R, ofault *F, const hs_model_desc *m, const hs_run_params *p, uint32_t r, const hs_outputs *out)
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

static void lfo_finish(orun *R, ofault *F)
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

int hs_fault_oracle_run_linked(uint32_t n_parts, const hs_model_desc *const *models, const hs_run_params *const *params,
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
    ofault *F = (ofault *)calloc(n_parts, sizeof(ofault));
    uint64_t *lat_draws = (uint64_t *)calloc(n_streams ? n_streams : 1, sizeof(uint64_t));
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t g = params[0]->replica_index_base + r;
        const uint64_t seed = cseed + (uint64_t)g * cseed_stride;
        const uint32_t rid = crid_base + g * crid_stride;
        uint64_t loss_draws = 0, n_del = 0, n_lost = 0;
        memset(lat_draws, 0, (n_streams ? n_streams : 1) * sizeof(uint64_t));
        for (uint32_t q = 0; q < n_parts; ++q) {
            lfo_init(&R[q], &F[q], models[q], params[q], r, outs[q]);
            R[q].outbox_cap = models[q]->outbox_cap;
            R[q].outbox = (hs_xevent *)calloc(R[q].outbox_cap ? R[q].outbox_cap : 1, sizeof(hs_xevent));
        }
        for (uint32_t w = 0; w < n_windows; ++w) {
            for (uint32_t q = 0; q < n_parts; ++q) fo_until(&R[q], &F[q], window_ends[w], -1);     /* 1. EXECUTE */
            for (uint32_t q = 0; q < n_parts; ++q) {                                                 /* 2. EXCHANGE */
                for (uint32_t k = 0; k < R[q].outbox_n; ++k) {
                    const hs_xevent *x = &R[q].outbox[k];
                    const hs_entity_desc *rem = &models[q]->entities[x->ent];
                    const hs_link_desc *lk = &links[q][rem->i0];
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
        for (uint32_t q = 0; q < n_parts; ++q) { free(R[q].outbox); lfo_finish(&R[q], &F[q]); }
        if (delivered) delivered[r] = n_del;
        if (lost) lost[r] = n_lost;
    }
    free(lat_draws); free(F); free(R);
    return HS_OK;
}
