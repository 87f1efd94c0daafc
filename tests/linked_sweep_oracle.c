/* linked_sweep_oracle.c -- the linked fault oracle (tests/linked_fault_oracle.c) for a linked run whose replicas are
 * sweep cells.  TEST INFRASTRUCTURE ONLY.
 *
 * hs_cells_oracle_run_linked is hs_fault_oracle_run_linked with
 *   - the partitions' cell overrides (hs_model_desc.cell_d0 / cell_i0, applied by orun_init from the replica's global
 *     index and params->replicas_per_cell),
 *   - the coordinator's per-cell link table links[q][cell * n_links[q] + k] (hs_coordinator_exchange_cells): replica g
 *     sends through row (g / replicas_per_cell) % n_cells, one loss draw only when its cell's loss is > 0,
 *   - the coordinator's seed and replica-word strides.
 * A model without FAULT rows runs as hs_oracle_run_linked runs it.
 * Built by tests/linked_sweep_lib.py into a temporary directory. */
#include "linked_fault_oracle.c"

int hs_cells_oracle_run_linked(uint32_t n_parts, const hs_model_desc *const *models, const hs_run_params *const *params,
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
        for (uint32_t q = 0; q < n_parts; ++q) { free(R[q].outbox); lfo_finish(&R[q], &F[q]); }
        if (delivered) delivered[r] = n_del;
        if (lost) lost[r] = n_lost;
    }
    free(lat_draws); free(F); free(R);
    return HS_OK;
}
