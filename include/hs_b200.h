/* hs_b200.h -- C-ABI of the H100 discrete-event engine (libhs_b200.so).
 *
 * The reference (adamfilli/happy-simulator) is pure Python and has NO FFI or
 * plugin registry for its run loop (SURVEY.md section 8(b)): the boundary it
 * offers is the Python object protocol
 *     Simulation(sources=, entities=, end_time=|duration=).run() -> SimulationSummary
 *     (happysimulator/core/simulation.py:66-76,230-288)
 *     ParallelRunner.run_replicas(build_fn, n, base_seed)
 *     (happysimulator/parallel/runner.py:115-142)
 * with results read back off the entity objects.  The entry points below are
 * what a ctypes binding of that boundary needs: upload a flattened model
 * (the object graph Simulation.__init__ receives), run N replicas of
 * Simulation.run()'s pop-invoke-push loop on the device, read per-replica
 * summaries / entity statistics / event records back.  Plain pointers and
 * sizes only; no torch types.  Every function returns 0 on success or a
 * negative hs_status; hs_last_error() gives the message of the calling
 * thread's last failure.  One host thread per engine handle.
 *
 * The same structs are the input/output format of the CPU oracle
 * (oracle/hs_oracle.c), so parity tests feed identical bytes to both sides.
 */
#ifndef HS_B200_H
#define HS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HS_ABI_VERSION 7u

typedef enum hs_status {
    HS_OK = 0,
    HS_ERR_INVALID = -1,     /* bad argument / unsupported model             */
    HS_ERR_CUDA = -2,        /* CUDA runtime failure (message has details)   */
    HS_ERR_NO_DEVICE = -3,   /* no CUDA device: the engine never falls back  */
    HS_ERR_STATE = -4,       /* call out of order (e.g. run before upload)   */
    HS_ERR_OVERFLOW = -5     /* a replica overflowed a fixed-size structure  */
} hs_status;

/* ---- model ------------------------------------------------------------- */

/* Entity kinds: the reference classes the engine lowers. */
enum {
    HS_ENT_SOURCE = 1,   /* load/source.py:92  Source (+SimpleEventProvider, ArrivalTimeProvider) */
    HS_ENT_SERVER = 2,   /* components/server/server.py:43 Server = Queue + QueueDriver + worker    */
    HS_ENT_SINK = 3,     /* components/common.py:18 Sink                                            */
    HS_ENT_COUNTER = 4,  /* components/common.py:79 Counter                                         */
    HS_ENT_LB = 5,       /* components/load_balancer/load_balancer.py:60 LoadBalancer               */
    HS_ENT_PROBE = 6,    /* instrumentation/probe.py:81 Probe's measurement callback (the Probe's own
                            ticking is a SOURCE row with a constant profile on the general path)     */
    HS_ENT_SKETCH = 7,   /* components/sketching/sketch_collector.py:24 SketchCollector over a HyperLogLog
                            (sketching/hyperloglog.py:43) or CountMinSketch (count_min_sketch.py:52) whose
                            value_extractor reads the request's routing key                           */
    HS_ENT_CACHE_SERVER = 8, /* examples/load-balancing/common.py:100-275 CachingServer: a QueuedResource without a
                            concurrency limit (Entity.has_capacity() is True) whose generator yields the cache-read
                            latency, on a miss the datastore latency, then the processing latency; one TTL cache
                            entry per customer key (TTLEviction, components/datastore/eviction_policies.py:154-226).
                            i0 = number of key slots K (keys 0..K-1; a request without a key uses slot K),
                            i1 = HS_Q_*, i2 / i3 = int(cache_read_latency_s * 1e9) / int(processing_latency_s * 1e9),
                            l0 = int(datastore_read_latency_s * 1e9), d0 = cache TTL (s), target = -1 (the generator
                            returns []).  The cache must be larger than the key population: the example raises
                            FrozenInstanceError on its first eviction (common.py:264), so eviction is not a
                            behaviour to reproduce and the lowering rejects such models.  Per-replica state: K + 1
                            insertion times (seconds; 0 = not cached), in the hs_outputs.sketches region.
                            hs_entity_stats: c0 accepted, c1 dropped, c2 requests_processed, c3 cache_misses,
                            f0 cache_hits, f1 cache_size (as doubles)                                   */
    HS_ENT_FAULT = 10,   /* one event of a node fault (faults/node_faults.py:16-128 CrashNode, PauseNode): an Event.once
                            aimed at a CallbackEntity that sets (crash, pause) or clears (restart, resume) `_crashed` on
                            the entity it names.  target = that entity, l0 = the event's time in ns (Instant.from_seconds),
                            i1 = 1 set / 0 clear, i2 = 1 if its FaultHandle was cancelled before the run, i3 = its
                            bootstrap sort index (global counter: sources, then probes, then the faults in schedule order;
                            in a linked partition the counter of that partition's own Simulation).
                            While an entity's flag is set, Event.invoke (core/event.py:261-262) drops the events aimed at it
                            -- counted and clock-moving, but neither handler nor completion hooks run: SOURCE_TICK (the
                            source is silent from then on), REQ_ENQUEUE, REQ_SINK, REQ_COUNTER, REQ_SKETCH, REQ_LB,
                            LB_RESPONSE.  hs_entity_stats: c0 = fired, c1 = popped while cancelled (events_cancelled,
                            core/simulation.py:475-477: not processed, the clock does not move).  A fault cannot target a
                            REMOTE row, and it sits next to REMOTE rows only in a model uploaded with
                            hs_partition_upload; the lane engine does not run them                          */
    HS_ENT_REMOTE = 9    /* stand-in for an entity that lives in ANOTHER partition of a ParallelSimulation
                            (parallel/simulation.py:31, parallel/routing.py:17-63): an event whose target is this row
                            is never scheduled here -- the partition's router puts it, with its send time, into the
                            partition's outbox, and the coordinator delivers it at the next window barrier
                            (parallel/coordinator.py:182-227).  i0 = slot (0..15) of the outgoing link in the hs_link_desc
                            array handed to hs_coordinator_exchange, i1 = the entity's id in the destination
                            partition's model.  hs_entity_stats: c0 = events sent through it                 */
};
/* Sketch algorithms of a SKETCH row.  Both hash the item with SHA-256 (hyperloglog.py:128-135,
 * count_min_sketch.py:136-155); the items are the routing keys 0..population-1, so the host evaluates
 * the hashes once per key (hs_model_desc.sketch_tables) and the device only indexes. */
enum { HS_SK_HLL = 1, HS_SK_CMS = 2,
       HS_SK_BLOOM = 3,   /* sketching/bloom_filter.py:57 BloomFilter (bit positions per key on the host)      */
       HS_SK_TOPK = 4,    /* sketching/topk.py:37 TopK, Space-Saving (no hashing: pure counter bookkeeping)     */
       HS_SK_TDIGEST = 5,   /* sketching/tdigest.py:47 TDigest behind components/sketching/quantile_estimator.py:35;
                             the value is the request's latency in seconds (Sink's, common.py:39-41)       */
       HS_SK_RESERVOIR = 6 }; /* sketching/reservoir.py:30 ReservoirSampler (Algorithm R on its own MT19937): i2 = size,
                             i1 = offset in sketch_tables of the generator state it starts from (mt[624], index) */
/* Probe metrics (getattr(target, metric), probe.py:55-62). */
enum { HS_METRIC_DEPTH = 0, HS_METRIC_ACTIVE_REQUESTS = 1, HS_METRIC_UTILIZATION = 2, HS_METRIC_AVAILABLE_CAPACITY = 3,
       HS_METRIC_STATS_ACCEPTED = 4, HS_METRIC_STATS_DROPPED = 5, HS_METRIC_EVENTS_RECEIVED = 6, HS_METRIC_TOTAL = 7,
       HS_METRIC_GENERATED_COUNT = 8 };
enum { HS_ARR_CONSTANT = 0, HS_ARR_POISSON = 1 };       /* load/providers/{constant,poisson}_arrival.py */
enum { HS_SVC_CONSTANT = 0, HS_SVC_EXPONENTIAL = 1 };   /* distributions/{constant,exponential}.py      */
enum { HS_Q_FIFO = 0, HS_Q_LIFO = 1,                   /* components/queue_policy.py:75,117            */
       HS_Q_PRIORITY = 2 };  /* queue_policy.py:189-287 PriorityQueue(key=happysim_b200.PriorityByKey(values)): pops the
                                smallest (values[routing key], insertion order); SERVER rows only, see hs_entity_desc.i3 */
enum { HS_LB_ROUND_ROBIN = 0, HS_LB_KEY_TABLE = 1 };    /* strategies.py:50 RoundRobin, :336 ConsistentHash
                                                           (ring lookup precomputed per key on the host) */

/* Processed-event kinds (what Simulation._execute_until pops; SURVEY.md 3.3). */
enum {
    HS_EV_SOURCE_TICK = 0,  /* SourceEvent -> Source                 load/source.py:142           */
    HS_EV_REQ_LB = 1,       /* Request -> LoadBalancer               load_balancer.py:347         */
    HS_EV_REQ_ENQUEUE = 2,  /* Request -> Server (Queue enqueue)     queue.py:122                 */
    HS_EV_NOTIFY = 3,       /* QueueNotifyEvent -> driver            queue_driver.py:92           */
    HS_EV_POLL = 4,         /* QueuePollEvent -> queue               queue.py:149                 */
    HS_EV_DELIVER = 5,      /* QueueDeliverEvent -> driver           queue_driver.py:66           */
    HS_EV_REQ_WORKER = 6,   /* Request -> worker (service start)     server/server.py:202         */
    HS_EV_CONTINUATION = 7, /* ProcessContinuation (service end)     core/event.py:465            */
    HS_EV_REQ_SINK = 8,     /* Request -> Sink                       common.py:36                 */
    HS_EV_LB_RESPONSE = 9,  /* _lb_response -> LoadBalancer          load_balancer.py:435         */
    HS_EV_REQ_COUNTER = 10, /* Request -> Counter                    common.py:92                 */
    HS_EV_PROBE = 11,       /* probe_event -> measurement callback   instrumentation/probe.py:51  */
    HS_EV_REQ_SKETCH = 12,  /* Request -> SketchCollector            sketch_collector.py:79       */
    HS_EV_FAULT = 13        /* fault callback (set / clear _crashed) node_faults.py:41-128; entity = the FAULT row */
};

typedef struct hs_entity_desc {
    int32_t kind;      /* HS_ENT_*                                                              */
    int32_t target;    /* SOURCE: entity receiving payloads; SERVER: downstream or -1; PROBE: measured entity */
    int32_t i0;        /* SOURCE: HS_ARR_*; SERVER: concurrency (FixedConcurrency); LB: HS_LB_*; PROBE: HS_METRIC_* */
    int32_t i1;        /* SOURCE: key population (0 = no routing key); SERVER: HS_Q_* (CACHE_SERVER: FIFO or LIFO);
                          LB: offset of its backend list in hs_model_desc.backends;
                          SKETCH: offset of its table in hs_model_desc.sketch_tables            */
    int32_t i2;        /* SOURCE: routing-key distribution: 0 = uniform (distributions/uniform.py:57), k > 0 = Zipf with
                          the cumulative probabilities key_cdf[k - 1 .. k - 1 + i1) (distributions/zipf.py:96-123);
                          SERVER: HS_SVC_*; LB: number of backends; SKETCH: HLL precision p | CMS depth | BLOOM num_hashes | TOPK k
                          | TDIGEST buffer size int(compression * 2), tdigest.py:88 */
    int32_t i3;        /* SOURCE: 0 = ConstantRateProfile(d0); k > 0 = profiles[k - 1] (non-constant
                          rate profile, general arrival path); SKETCH: CMS width | BLOOM size_bits
                          | TDIGEST centroid capacity (>= 2 x buffer size);
                          SERVER with HS_Q_PRIORITY: 1 + offset in hs_model_desc.profile_table of its priority table, one
                          double per routing key (priority of key k = table[k]; no NaN), covering the key population of
                          every SOURCE row; every SOURCE row that sends requests (all but a Probe's ticking) must draw
                          keys -- a request without one has no priority, the reference's key raises.  The lane engine
                          does not run such a model.  Other SERVER rows: 0; others: reserved, 0 */
    int64_t l0;        /* SOURCE: stop_after in ns or -1; SERVER: queue capacity or -1 (= inf);
                          SKETCH: key population K = row stride of its table in sketch_tables; 0 = no per-key
                          table: the device evaluates the SHA-256 hashes per event (any key population) and
                          the table holds only the seed words, see hs_model_desc.sketch_tables       */
    double d0;         /* SOURCE: rate (events/s); SERVER: mean / constant service time (s);
                          SKETCH/TDIGEST: compression                                           */
    double d1;         /* reserved, 0                                                           */
} hs_entity_desc;      /* 48 bytes */

typedef struct hs_model_desc {
    uint32_t abi_version;          /* HS_ABI_VERSION */
    uint32_t n_entities;
    const hs_entity_desc *entities;
    uint32_t n_backends;           /* total length of backends[]                               */
    uint32_t key_population;       /* length of key_table[] (0 if unused)                      */
    const int32_t *backends;       /* entity ids, LB backend lists concatenated                */
    const int32_t *key_table;      /* routing key -> index into the LB's backend list          */
    /* Parameter sweep ("cells"): replica r belongs to cell r / replicas_per_cell; a cell
     * overrides d0 / i0 of every entity.  NULL = no override.                                 */
    uint32_t n_cells;
    uint32_t outbox_cap;           /* linked partitions: cross-partition events one replica can emit per window
                                      (0: the model has no REMOTE rows)                                        */
    const double *cell_d0;         /* [n_cells][n_entities] or NULL */
    const int32_t *cell_i0;        /* [n_cells][n_entities] or NULL */
    /* Non-constant rate profiles (load/profile.py LinearRampProfile, SpikeProfile): arrival times
     * come from the reference's adaptive-Simpson + Brent path (arrival_time_provider.py:84-144). */
    uint32_t n_profiles;
    uint32_t inbox_cap;            /* linked partitions: cross-partition events one replica can receive per
                                      barrier (0: no link ends in this partition)                            */
    const struct hs_profile_desc *profiles;   /* 40 bytes each, see below */
    /* Per-key hash results of the SKETCH rows (row i0/i1/i2/i3/l0: algorithm, table offset, p | depth,
     * CMS width, K).  HLL: [2][K] = register index (hash >> (64 - p)) and run length (leading zeros of
     * the remaining bits + 1) of key k, hyperloglog.py:156-165.  CMS: [depth][K] = column of key k in
     * each row, count_min_sketch.py:145-155.  BLOOM: [num_hashes][K] = bit index (h1 + i h2) mod size_bits of
     * key k for hash i, bloom_filter.py:147-160.  TOPK: no table.
     * A row with K = 0 hashes on the device (csrc/hs_sketch.h: SHA-256 of the packed seed and repr(key)); its
     * table is then the seed as (lo, hi) int32 words -- HLL, BLOOM: the sketch's seed; CMS: the depth row
     * seeds sha256(pack(">QQ", seed, row))[:8] (count_min_sketch.py:136-143). */
    uint32_t n_sketch_table;       /* total length of sketch_tables[]                          */
    uint32_t n_key_cdf;            /* total length of key_cdf[]                                */
    const int32_t *sketch_tables;
    /* ZipfDistribution._cum_probs of the sources whose keys are Zipf distributed (zipf.py:96-110), as the
     * host computed them; a key is bisect_left(cum_probs, u) clamped to the last index (zipf.py:112-123). */
    const double *key_cdf;
    /* Tables of the piecewise-constant (STEP) rate profiles: for a profile with n breakpoints, n ascending
     * breakpoints (seconds) followed by n + 1 rates; rate(t) = rates[#{breakpoints <= t}].  A user-defined
     * Profile.get_rate that is a step function (examples/queuing/m_m_1_queue.py:104-169) lowers to one.
     * The priority tables of HS_Q_PRIORITY servers (one double per routing key, see hs_entity_desc.i3) are appended
     * to the same array. */
    const double *profile_table;
    uint64_t n_profile_table;      /* total length of profile_table[]                          */
} hs_model_desc;

enum { HS_PROF_CONSTANT = 0, HS_PROF_LINEAR_RAMP = 1, HS_PROF_SPIKE = 2, HS_PROF_STEP = 3 };
typedef struct hs_profile_desc {
    int32_t kind;      /* HS_PROF_*                                                          */
    int32_t pad;
    double p[4];       /* CONSTANT: rate | LINEAR_RAMP: duration_s, start_rate, end_rate
                          | SPIKE: baseline_rate, spike_rate, warmup_s, spike_duration_s
                          | STEP: offset of its table in profile_table, number of breakpoints n,
                            p[2] = the ADDRESS of that table as a bit pattern (filled in by whoever
                            evaluates the profile: the engine writes the device address into its copy,
                            the host layer the host address for the CPU oracle), p[3] unused          */
} hs_profile_desc;     /* 40 bytes */

/* ---- run --------------------------------------------------------------- */

typedef struct hs_run_params {
    uint64_t seed;             /* Philox key of replica r = seed + r * seed_stride             */
    uint64_t seed_stride;      /* 1 mirrors ParallelRunner (base_seed + i), 0 for ensembles    */
    uint32_t rid_base;         /* Philox replica word of replica r = rid_base + r * rid_stride */
    uint32_t rid_stride;
    int64_t end_ns;            /* Simulation end_time; the loop processes while now <= end_ns  */
    uint32_t n_replicas;       /* replicas run by THIS call                                    */
    uint32_t replica_index_base; /* global index of this call's replica 0 (multi-GPU shards)   */
    uint32_t replicas_per_cell;  /* cell = global index / replicas_per_cell (>=1)              */
    /* Flight-recorder rings, per replica: item i of a stream lives at slot i % cap, so the
     * buffers hold the LAST cap items (everything when cap >= count).  Every item is written
     * to its ring in device memory: 16 B per processed event (streamed as whole 128-byte lines), 16 B per
     * Sink sample and 8 B per service start (through L2, which completes their lines).     */
    uint32_t record_cap;       /* event-record ring entries per replica (0 = no trace)         */
    uint32_t sample_cap;       /* Sink-sample ring entries per replica                         */
    uint32_t service_cap;      /* service-time ring entries per replica                        */
    uint32_t queue_ring;       /* device queue ring entries per server (power of two), 0 = default */
    uint32_t engine;           /* 0 auto, 1 warp engine (general), 2 lane engine (single FIFO / LIFO server), 3 thread engine (general) */
    /* Windowed execution (reference: Simulation._run_window, core/simulation.py:527-541):
     * when 0 <= window_end_ns < end_ns the call pauses every replica before the first
     * event later than window_end_ns and keeps its state on the device; a following
     * call with resume = 1 continues from there.  The processed-event sequence of a
     * run cut into windows is identical to the uncut run.  window_end_ns < 0: run to
     * end_ns. */
    int64_t window_end_ns;
    uint32_t resume;           /* 1 = continue the replicas of the previous call          */
    uint32_t flags;            /* HS_RUN_* bits                                           */
    int64_t max_events;        /* safety valve: a replica stops (HS_ST_EVENT_LIMIT) once it has
                                  processed this many events in total; 0 = unlimited.  A model
                                  whose clock cannot advance (e.g. a constant source faster than
                                  1 event/ns) never terminates in the reference either.        */
} hs_run_params;

#define HS_RUN_ORDER_HASH 1u   /* maintain hs_replica_summary.order_hash (off: hash = 0)  */
#define HS_RUN_HISTOGRAM 2u    /* per-replica 64-bin latency histogram of all Sink events  */
#define HS_RUN_LINKED 4u       /* a window of a linked partition (hs_coordinator_*): with resume = 1, replicas that
                                  had finished (clock past the previous end_ns, or nothing pending) run on -- end_ns
                                  is the new window end and the barrier may have delivered events               */
#define HS_HISTOGRAM_BINS 64   /* log-spaced over integer ns, see hs_latency_bin()         */

/* Replica status bits. */
#define HS_ST_QUEUE_OVERFLOW 1u   /* a server's device queue ring filled up  */
#define HS_ST_FEL_OVERFLOW 2u     /* future-event list slots exhausted       */
#define HS_ST_REJECT_PATH 4u      /* Server acquire failed (server.py:223)   */
#define HS_ST_TRACE_EXHAUSTED 8u  /* ran out of externally supplied draws    */
#define HS_ST_EVENT_LIMIT 16u     /* hs_run_params.max_events reached        */
#define HS_ST_SKETCH_OVERFLOW 32u /* a TDigest outgrew its centroid capacity */
#define HS_ST_LINK_OVERFLOW 64u   /* a partition's outbox or inbox filled up */
#define HS_ST_LINK_TIE 128u       /* linked partitions: an event delivered over a link tied with another event on BOTH time
                                     and sort index (the indices come from different partitions' counters).  The reference
                                     orders such a pair by the accident of heapq's array layout; the engines order it by
                                     their own heap's, so this replica's event order may differ from the reference's      */
#define HS_ST_FAULT_TIE 256u      /* an event created during the run, or delivered over a link, tied with a pending FAULT
                                     event on both time and sort index (the fault's index comes from the bootstrap counter,
                                     the other's from the run's or from the sending partition's):
                                     heapq orders such a pair by its array layout, the engines by their own heap's, so this
                                     replica's event order may differ from the reference's                               */
#define HS_ST_BUCKET_OVERFLOW 512u /* bucket percentiles (hs_set_bucket_percentiles): a bucket held more samples than the
                                     sample capacity; its p50 / p99 are NaN, its record's count is exact             */

typedef struct hs_replica_summary {
    int64_t events_processed;  /* SimulationSummary.total_events_processed (simulation.py:553) */
    int64_t final_time_ns;     /* clock after the last processed event (simulation.py:503)     */
    uint64_t order_hash;       /* hs_hash_step over every processed event, in order            */
    uint64_t next_sort_index;  /* value of the per-heap creation counter at the end            */
    int64_t n_sink_samples;    /* Sink samples produced (all sinks); ring position = n % cap   */
    int64_t n_service_samples; /* service starts (Server._service_times appends)               */
    int32_t heap_left;         /* events still pending (linked partitions: incl. delivered, not yet taken) */
    uint32_t status;           /* HS_ST_* bits, 0 = clean                                      */
} hs_replica_summary;          /* 56 bytes */

typedef struct hs_entity_stats {
    int64_t c0; /* SOURCE generated_count | SERVER stats_accepted | SINK events_received
                   | COUNTER total | LB requests_received | PROBE samples taken
                   | SKETCH events_processed                                                   */
    int64_t c1; /* SOURCE payloads created | SERVER stats_dropped | LB requests_forwarded
                   | SKETCH item_count (requests that carried a key)                           */
    int64_t c2; /* SERVER requests_completed | LB in-flight entries left                        */
    int64_t c3; /* SERVER requests_rejected | SERVER (after run) -- ; LB responses handled      */
    double f0;  /* SERVER total_service_time (sequential +=) | SINK sum(latencies_s) as CPython's
                   float sum() computes it (Neumaier-compensated), so f0 / c0 == average_latency() */
    double f1;  /* SINK sum of squared latencies                                                */
    double f2;  /* SINK min latency (+inf if none)                                              */
    double f3;  /* SINK max latency (-inf if none)                                              */
} hs_entity_stats;             /* 64 bytes */

typedef struct hs_event_record {   /* 16 bytes per processed event (SURVEY.md 8(d))            */
    int64_t time_ns;
    uint32_t sort_index;           /* low 32 bits of Event._sort_index                         */
    uint8_t kind;                  /* HS_EV_*                                                  */
    uint8_t pad;
    uint16_t entity;               /* entity id (hidden queue/driver/worker -> their Server)    */
} hs_event_record;

typedef struct hs_sink_sample {    /* Sink.completion_times[i], Sink.latencies_s[i]            */
    int64_t completion_ns;
    double latency_s;
} hs_sink_sample;

typedef struct hs_outputs {        /* caller-owned HOST buffers; any pointer may be NULL        */
    hs_replica_summary *summaries; /* [n_replicas]                                             */
    hs_entity_stats *entity_stats; /* [n_replicas][n_entities]                                 */
    hs_event_record *records;      /* [n_replicas][record_cap] ring, slot = event number % cap */
    hs_sink_sample *sink_samples;  /* [n_replicas][sample_cap], all sinks, arrival order       */
    double *service_samples;       /* [n_replicas][service_cap], service-start order           */
    uint32_t *histograms;          /* [n_replicas][HS_HISTOGRAM_BINS] (HS_RUN_HISTOGRAM)        */
    uint8_t *sketches;             /* [n_replicas][hs_sketch_layout().total]: every SKETCH row's state,
                                      HLL: uint8 registers[2^p]; CMS: uint32 counters[depth][width];
                                      BLOOM: uint64 words[ceil(size_bits / 64)]; TOPK: uint32 n, pad[3], then
                                      k x {int32 item, uint32 count, uint32 error} in dict (insertion) order;
                                      TDIGEST: {uint32 n_centroids, n_buffer; int64 total; double min, max},
                                      capacity x {double mean; int64 count}, buffer double[buffer size]       */
} hs_outputs;

/* Ensemble totals: what the single end-of-run NCCL allreduce carries (SURVEY.md 8(e)).
 * Sums are over replicas; extrema are min/max.  Fixed layout so ranks can reduce it as
 * int64[HS_TOTALS_I64] (sum), double[HS_TOTALS_F64_SUM] (sum) and two extrema (min, max). */
#define HS_TOTALS_I64 8
#define HS_TOTALS_F64_SUM 3
typedef struct hs_totals {
    int64_t i[HS_TOTALS_I64];  /* 0 events_processed, 1 sink events, 2 server completions,
                                  3 source ticks, 4 dropped, 5 replicas, 6 replicas with
                                  status != 0, 7 sum of final_time_ns / 1000 (us)              */
    double fsum[HS_TOTALS_F64_SUM]; /* 0 sum latency, 1 sum latency^2, 2 sum service time      */
    double fmin;               /* min sink latency */
    double fmax;               /* max sink latency */
} hs_totals;

/* Per-cell aggregates of a parameter sweep (BASELINE configs[4]: the vector that is all-reduced
 * per (c, rho) cell): the ensemble totals restricted to the replicas of one cell, plus the cell's
 * latency histogram (sum over its replicas; zeros unless HS_RUN_HISTOGRAM was set). */
typedef struct hs_cell_totals {
    hs_totals totals;
    uint64_t histogram[HS_HISTOGRAM_BINS];
} hs_cell_totals;

/* Time buckets (hs_set_buckets): the reference's Data.bucket(window_s) (instrumentation/data.py:127-158) of every
 * replica's Sink / LatencyTracker / ThroughputTracker / Probe samples, reduced on the device as the samples arrive.
 * The bucketed rows are the model's SINK and PROBE rows in entity order (row b = the b-th of them).  A sample at t ns
 * with value v (a Sink's latency in seconds, a Probe's metric) goes to bucket k = floor((t / 1e9) / width_s), both
 * divisions correctly rounded, as math.floor(Instant.to_seconds() / window_s) computes it. */
typedef struct hs_bucket {         /* one bucket of one row of one replica, 32 bytes                        */
    int64_t count;                 /* samples in the bucket (0: the bucket is empty, Data.bucket omits it)   */
    double sum, comp;              /* sum(values) as CPython's float sum() computes it: sum + comp (Neumaier) */
    double max;                    /* max(values); meaningless when count == 0                              */
} hs_bucket;

/* One bucket of one row over the replicas of one sweep cell, 48 bytes.  Summed in a fixed order (replicas in index
 * order within slices of at most 256 that do not cross a cell boundary, then the slices in index order), with no
 * atomics: repeated runs give the same bits whichever engine ran the replicas. */
typedef struct hs_bucket_total {
    int64_t replicas;              /* replicas with at least one sample in the bucket                         */
    int64_t count;                 /* sum of their counts                                                     */
    double sum;                    /* sum of their bucket sums (sum + comp each)                              */
    double mean_sum, mean_sq_sum;  /* sum of their bucket means (sum / count) and of the squared means        */
    double max;                    /* max of their maxes (-inf if replicas == 0)                              */
} hs_bucket_total;

/* The p50 / p99 of one bucket of one row over the replicas of one sweep cell, 32 bytes, in the order and the slices
 * of hs_bucket_total.  Only replicas with at least one sample in the bucket contribute: their number is that
 * hs_bucket_total's `replicas`. */
typedef struct hs_bucket_pct_total {
    double p50_sum, p50_sq_sum;    /* sum of their bucket p50s and of the squared p50s                         */
    double p99_sum, p99_sq_sum;    /* the same for p99                                                         */
} hs_bucket_pct_total;

/* ---- entry points ------------------------------------------------------ */

typedef struct hs_engine hs_engine;

/* Library / ABI version (HS_ABI_VERSION of the build). */
uint32_t hs_version(void);

/* Message of the calling thread's last error; returns its length. */
int hs_last_error(char *buf, int len);

/* Create an engine on CUDA device `device`, launching on `stream` (a cudaStream_t
 * cast to void*, NULL = a private non-blocking stream).  Replaces
 * Simulation.__init__'s heap/clock construction (core/simulation.py:93-106).
 * Fails with HS_ERR_NO_DEVICE when no GPU is present: there is no CPU path. */
int hs_engine_create(int device, void *stream, hs_engine **out);
int hs_engine_destroy(hs_engine *e);

/* Validate and upload the flattened model (what Simulation.__init__ receives
 * as sources=/entities=, core/simulation.py:95-102). */
int hs_model_upload(hs_engine *e, const hs_model_desc *model);

/* Validate a model without a device (used by host-side tests). */
int hs_model_validate(const hs_model_desc *model);

/* hs_model_upload / hs_model_validate for one partition of a linked run (ParallelSimulation with PartitionLinks,
 * parallel/simulation.py:94-104): the partition's Simulation bootstraps its own fault schedule, so FAULT rows may sit
 * next to its REMOTE rows (a FAULT row still cannot target one).  A model uploaded with hs_model_upload that has
 * FAULT rows does not run as a linked partition (hs_run with outbox / inbox / HS_RUN_LINKED). */
int hs_partition_upload(hs_engine *e, const hs_model_desc *model);
int hs_partition_validate(const hs_model_desc *model);

/* Byte offsets of the SKETCH rows' state.  per_replica[i] / merged[i] = offset of entity i's state in
 * one replica's slice of hs_outputs.sketches / in the merged image (0 for other kinds); a replica's
 * slice is *total bytes, the merged image *merged_total.  The merged image applies the reference's
 * merge() contracts over the replicas of a run: HLL registers -> element-wise max (hyperloglog.py:
 * 203-226), uint8[2^p]; CMS counters -> element-wise sum (count_min_sketch.py:276-301), widened to
 * uint64[depth][width]; BLOOM words -> bitwise OR (bloom_filter.py:262-291).  TopK.merge (topk.py:216-258)
 * and TDigest.merge (tdigest.py:326-352) are order dependent and sequential: TOPK / TDIGEST rows have no
 * merged image (size 0), the host layer merges the per-replica states.  Needs no device. */
int hs_sketch_layout(const hs_model_desc *model, uint64_t *per_replica, uint64_t *merged,
                     uint64_t *total, uint64_t *merged_total);

/* Externally supplied draws ("stock generator" mode).  The reference draws arrival target
 * areas as -log(1 - numpy.random.random()) (load/providers/poisson_arrival.py:31) and service
 * samples as random.expovariate(lambda) (distributions/exponential.py:43) from two process-global
 * MT19937 streams that every consumer shares in call order.  The host can generate those two
 * streams with the very generators the reference uses and hand them over: replica r reads
 * arrival_targets[r * n_arrival + k] for the k-th Poisson draw made by ANY source and
 * service_samples[r * n_service + k] for the k-th exponential draw made by ANY server, in
 * simulation order.  Both arrays hold unit-rate exponential variates -log(1 - U) evaluated on the
 * host with the reference's libm; the consumer's own rate / lambda is applied on the device
 * (target / rate, and expovariate's  -log(1 - U) / lambd).  Everything downstream of the draw
 * (divisions, ns truncation) is the device's usual arithmetic, so a run reproduces the unmodified, stock-seeded reference bit for bit.
 * Buffers are copied to the device; pass NULL/0 to return to the Philox streams.  A replica that
 * runs out of draws stops with HS_ST_TRACE_EXHAUSTED. */
int hs_set_trace(hs_engine *e, const double *arrival_targets, uint64_t n_arrival,
                 const double *service_samples, uint64_t n_service, uint32_t n_replicas);

/* Simulation.run() for params->n_replicas replicas (core/simulation.py:230,
 * 449-505).  Asynchronous on the engine's stream; results stay on the device
 * until hs_read_outputs / hs_read_totals. */
int hs_run(hs_engine *e, const hs_run_params *params);

/* Wait for the stream; returns HS_ERR_CUDA on a device fault. */
int hs_sync(hs_engine *e);

/* Device milliseconds of the last hs_run's kernels (CUDA events on the engine stream). */
int hs_last_run_ms(hs_engine *e, float *ms);

/* Number of kernels hs_run launched since engine creation. */
int hs_launch_count(hs_engine *e, uint64_t *n);

/* Which compiled kernel the last hs_run launched, and its geometry.  The engines pick their kernel from the
 * model, the ensemble size and the device's SM count; this reports the choice without changing it. */
enum { HS_KERNEL_LANE = 1, HS_KERNEL_WARP = 2, HS_KERNEL_THREAD = 3, HS_KERNEL_THREAD_WIDE = 4 };
typedef struct hs_launch_info {
    uint32_t engine;               /* 1 warp, 2 lane, 3 thread (hs_run_params.engine after auto selection) */
    uint32_t kernel;               /* HS_KERNEL_* family */
    uint32_t flags;                /* template FLAGS of the launched instantiation (HS_LF_* / HS_WF_* of csrc/) */
    uint32_t lane_stride;          /* thread engine: lanes per replica (32 / replicas per warp); 1 otherwise */
    uint32_t heap_top;             /* thread engine: heap keys per replica held in shared memory; 0 otherwise */
    uint32_t grid, block;          /* blocks, threads per block */
    uint32_t smem;                 /* dynamic shared memory per block, bytes */
} hs_launch_info;      /* 32 bytes */
int hs_last_launch(hs_engine *e, hs_launch_info *out);

/* Copy results of the last run to caller-owned host buffers (synchronises). */
int hs_read_outputs(hs_engine *e, const hs_outputs *out);

/* Reduce the last run's per-replica results on the device and copy the totals
 * (SimulationSummary-level aggregates) to the host (synchronises). */
int hs_read_totals(hs_engine *e, hs_totals *out);

/* Reduce the last run's replicas per sweep cell (cell = global replica index /
 * replicas_per_cell, modulo n_cells) on the device and copy out[0..n_cells) to the host. */
int hs_read_cell_totals(hs_engine *e, hs_cell_totals *out, uint32_t n_cells);

/* Merge the last run's per-replica sketches on the device (layout: hs_sketch_layout's merged image)
 * and copy the image to the host; what a multi-GPU run all-reduces (max for HLL bytes, sum for CMS). */
int hs_read_sketches(hs_engine *e, void *merged, uint64_t merged_bytes);

/* ---- linked partitions (parallel/coordinator.py:28-227) --------------------------------------------
 * A ParallelSimulation with PartitionLinks is one engine per partition (each with the same replicas) plus one
 * coordinator.  Per window the host layer runs every partition with hs_run(end_ns = window end, resume = window > 0)
 * -- Simulation._run_window = _execute_until(window_end), core/simulation.py:527-541: the loop test is on the LAST
 * processed time, so a partition also processes its first event beyond the window end -- and then calls
 * hs_coordinator_exchange once per partition, in partition order (WindowedCoordinator._exchange_events walks the
 * outboxes in that order).  An event delivered earlier than the destination's clock is "time travel" and is
 * skipped, uncounted, exactly as the reference's loop skips it (core/simulation.py:479-489). */
typedef struct hs_xevent {        /* one cross-partition event, 40 bytes */
    int64_t time_ns;              /* outbox: send time (the sender's clock); inbox: arrival time            */
    uint64_t sort_index;          /* Event._sort_index, from the SENDER's per-heap counter (event_heap.py:48) */
    int64_t created_ns;           /* context["created_at"]                                                   */
    uint64_t aux;                 /* reserved (0)                                                            */
    int32_t key;                  /* context["metadata"]["client_id"], -1 if none                            */
    int32_t ent;                  /* outbox: the REMOTE row it was sent to; inbox: target entity id          */
} hs_xevent;

typedef struct hs_link_desc {     /* parallel/link.py:18 PartitionLink with a latency override               */
    int32_t latency_kind;         /* HS_SVC_CONSTANT | HS_SVC_EXPONENTIAL: event.time = send_time + sample()  */
    int32_t stream;               /* id of the latency OBJECT: links that share one object share its draws    */
    double latency_mean_s;
    double packet_loss;           /* in [0, 1): one coordinator draw per event when > 0 (coordinator.py:204)  */
} hs_link_desc;

typedef struct hs_coordinator hs_coordinator;
/* Per-replica coordinator state on `device`: the draw counters of the loss stream and of n_streams latency
 * streams, delivered / lost totals.  Philox key and replica word of replica r as in hs_run_params. */
int hs_coordinator_create(int device, void *cuda_stream, uint32_t n_replicas, uint32_t n_streams,
                          uint64_t seed, uint64_t seed_stride, uint32_t rid_base, uint32_t rid_stride,
                          uint32_t replica_index_base, hs_coordinator **out);
void hs_coordinator_destroy(hs_coordinator *c);
/* Drain src's outboxes: every event goes through its REMOTE row's link links[row.i0] (loss draw, then
 * time = send time + latency sample) into the inbox of dsts[row.i0] with target row.i1; the next hs_run of that
 * engine pushes its inbox into the replicas' heaps before the first pop (Simulation.schedule, :195-206). */
int hs_coordinator_exchange(hs_coordinator *c, hs_engine *src, uint32_t n_links, const hs_link_desc *links,
                            hs_engine *const *dsts);
/* hs_coordinator_exchange for a linked run whose replicas are sweep cells: links[cell][k], n_cells rows of n_links, and
 * replica g (= replica_index_base + r) sends through row (g / replicas_per_cell) % n_cells -- the cell the partitions'
 * hs_model_desc.cell_d0 / cell_i0 give it.  latency_mean_s and packet_loss may differ between the rows; latency_kind
 * and stream (which latency object a link draws from) must be equal in every row, and the destination dsts[k] is one
 * for all cells.  Each replica draws exactly as hs_coordinator_exchange with its row's values: a loss draw only when
 * its cell's packet_loss is > 0.  The table is kept on the device per source engine and copied again only when its
 * bytes change, so the windows of a run upload it once.  hs_coordinator_exchange is the one-cell case of the same
 * barrier. */
int hs_coordinator_exchange_cells(hs_coordinator *c, hs_engine *src, uint32_t n_links, uint32_t n_cells,
                                  uint32_t replicas_per_cell, const hs_link_desc *links, hs_engine *const *dsts);
/* The checks hs_coordinator_exchange_cells makes of links[n_cells][n_links], without a device: a valid latency kind,
 * latency_mean_s >= 0 and packet_loss in [0, 1) in every row, latency_kind and stream equal to row 0's. */
int hs_link_cells_validate(uint32_t n_links, uint32_t n_cells, const hs_link_desc *links);
/* per-replica totals since create ([n_replicas] each, any pointer may be NULL): events delivered into inboxes,
 * events lost on lossy links, events that found the destination's inbox full (a sizing error: raise inbox_cap) */
int hs_coordinator_read(hs_coordinator *c, uint64_t *delivered, uint64_t *lost, uint64_t *overflowed);
/* Copy the current outboxes / inboxes to the host: buf[n_replicas][cap], counts[n_replicas] (tests, debugging). */
int hs_read_outbox(hs_engine *e, hs_xevent *buf, uint32_t *counts);
int hs_read_inbox(hs_engine *e, hs_xevent *buf, uint32_t *counts);

/* Time buckets for the following hs_run calls: width_s > 0 seconds, n buckets per row and replica (n = 0: off, the
 * default).  Per replica the engine keeps [rows][n + 1] hs_bucket records: slot k < n is bucket k, slot n holds the
 * samples with an index >= n (only the one event a replica processes past end_ns can make one; its index is kept
 * separately).  hs_run refuses a bucketed run whose end time falls into bucket n or later (n * width_s must exceed
 * the end time), a run with recorder rings (record_cap, sample_cap or service_cap: buckets are the summary-mode
 * series; the rings stay the record-mode path), a window of a linked partition (HS_RUN_LINKED or a model with
 * REMOTE rows) whose model did not come through hs_partition_upload, and a resume whose bucket configuration differs
 * from the paused run's.  The windows of a linked run keep their buckets like those of a windowed run: every window
 * passes the same configuration, and the last one's records are the whole run's.  It checks the size of the records
 * against the free device memory before it allocates them. */
int hs_set_buckets(hs_engine *e, double width_s, uint32_t n);

/* Copy the last run's buckets: out[n_replicas][rows][n + 1] (see hs_set_buckets) and past_end[n_replicas][rows], the
 * index of the samples in slot n (valid where that slot's count > 0).  Either pointer may be NULL.  *rows (if not
 * NULL) receives the number of bucketed rows. */
int hs_read_buckets(hs_engine *e, hs_bucket *out, int64_t *past_end, uint32_t *rows);

/* Reduce the last run's buckets per sweep cell (cell = global replica index / replicas_per_cell, modulo n_cells, as
 * hs_read_cell_totals) on the device and copy out[n_cells][rows][n + 1] to the host.  Slot n aggregates the
 * past-end samples whatever their index. */
int hs_read_bucket_totals(hs_engine *e, hs_bucket_total *out, uint32_t n_cells);

/* Bucket percentiles for the following hs_run calls (sample_cap = 0: off, the default): besides its hs_bucket record
 * every bucket gets the reference's _percentile_sorted(sorted(values), 0.50) and (..., 0.99)
 * (instrumentation/data.py:197-210), bit for bit.  The engine holds the values of each row's current bucket, at most
 * sample_cap of them per row and replica, and selects the two order-statistic pairs when the row moves on and when a
 * launch ends.  A bucket with more than sample_cap samples gets NaN for both and sets HS_ST_BUCKET_OVERFLOW in its
 * replica's status; its record's count says what capacity a re-run needs.  hs_run refuses percentiles without
 * buckets (hs_set_buckets n > 0) and a resume whose capacity differs from the paused run's; its memory check covers
 * the value buffers and the percentile records. */
int hs_set_bucket_percentiles(hs_engine *e, uint32_t sample_cap);

/* Copy the last run's bucket percentiles: out[n_replicas][rows][n + 1][2], {p50, p99} per slot as hs_read_buckets
 * lays out the records (0, 0 for an empty bucket). */
int hs_read_bucket_percentiles(hs_engine *e, double *out);

/* Reduce the last run's bucket percentiles per sweep cell, as hs_read_bucket_totals reduces the records, and copy
 * out[n_cells][rows][n + 1] to the host. */
int hs_read_bucket_percentile_totals(hs_engine *e, hs_bucket_pct_total *out, uint32_t n_cells);

/* Device pointer/size of the last run's totals (for the NCCL allreduce done by
 * the host layer on torch.distributed; layout = hs_totals). */
int hs_totals_device_ptr(hs_engine *e, void **ptr);

#ifdef __cplusplus
}
#endif
#endif /* HS_B200_H */
