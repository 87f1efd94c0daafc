/* hs_kernel_params.cuh -- the run parameters and output pointers every engine kernel (lane, warp, thread) takes,
 * filled once per hs_run by the host.  What the engines' models look like differs (hs_lane_model, hs_warp_model). */
#ifndef HS_KERNEL_PARAMS_CUH
#define HS_KERNEL_PARAMS_CUH

#include "../../include/hs_b200.h"

struct hs_kernel_run {
    uint64_t seed, seed_stride;
    uint32_t rid_base, rid_stride;
    int64_t end_ns, window_end_ns;
    uint32_t n_replicas, index_base, replicas_per_cell;
    uint32_t record_cap, sample_cap, service_cap, ring, resume;
    int64_t max_events;                     /* INT64_MAX = unlimited */
    const double *trace_arr, *trace_svc;    /* externally supplied draws (hs_set_trace) or NULL */
    uint64_t n_trace_arr, n_trace_svc;
    /* thread engine only */
    uint32_t linked;                /* HS_RUN_LINKED: a window of a linked partition -- finished replicas continue */
    uint32_t lane_stride;           /* lanes per replica (1, 2, 4 ... 32) */
    uint32_t heap_top;              /* number of heap keys (whole top levels: 0, 5, 21, 85 or 341 for arity 4) kept in
                                       shared memory during a launch, [key][replica column] */
};

struct hs_kernel_out {
    hs_replica_summary *summaries;
    hs_entity_stats *stats;
    hs_event_record *records;
    hs_sink_sample *samples;
    double *service;
    uint32_t *hist;                 /* [replica][HS_HIST_BINS] or NULL */
    uint8_t *sketch;                /* [replica][sk_total] (warp and thread engines) */
    hs_xevent *outbox; uint32_t *outbox_n;   /* [replica][outbox_cap], entries used (linked partitions) */
    hs_xevent *inbox; uint32_t *inbox_n;     /* [replica][inbox_cap], entries waiting to be scheduled   */
};

#endif /* HS_KERNEL_PARAMS_CUH */
