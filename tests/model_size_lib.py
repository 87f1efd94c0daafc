"""The general engines' layout rules restated in Python, and the models whose sizes put them at each layout.

The warp engine (launch_warp and general_setup, csrc/hs_engine.cu) stages one replica block per warp in shared
memory: the block's size decides the warps per CTA, whether the model tables are copied into shared memory, and
whether the model runs at all.  The thread engine (launch_thread) gives every entity its own payload slot when every
entity has at most one pending future event and there are no more entities than future-event slots.
tests/test_model_sizes.py checks these restatements against hand-computed values, tests/test_gpu_model_sizes.py
against Engine.last_launch(), so a change to a sizing rule fails there instead of silently moving the coverage.
Test infrastructure."""
import numpy as np

import happysim_b200 as hs
from happysim_b200 import _abi as A
from high_water_lib import HS_W_NCAP, fel_slots

WARP_HDR = 128                          # sizeof(hs_warp_hdr), csrc/hs_warp_engine.cuh
WENT = 96                               # sizeof(hs_went)
WNOW = 48                               # sizeof(hs_wnow)
MBAR = 16                               # the mbarrier slot in front of a warp's block
WARP_SMEM_MAX = 227 * 1024 - 1024       # HS_WARP_SMEM_MAX: dynamic shared memory of a warp-engine CTA
WARP_SMEM_BUDGET = 200 * 1024           # launch_warp: warps per CTA from half of this
SLOT_LIMIT = 65535                      # general_setup refuses S above this (16-bit slot ids)
ENTITY_LIMIT = 65535                    # hs_model_validate: n_entities in 1..65535 (16-bit entity ids)


def _ceil(x, unit):
    return (x + unit - 1) // unit * unit


def warp_block_bytes(model):
    """general_setup's replica block for the warp engine: header, entity rows, the future tier (S slots x 46 B,
    SoA, with the free-slot stack) rounded to 16 B, the now tier"""
    return WARP_HDR + model.n_entities * WENT + _ceil(fel_slots(model) * 46, 16) + HS_W_NCAP * WNOW


def warp_geometry(model):
    """launch_warp's layout: dict(per_warp, model_bytes, warps, smem), model_bytes = 0 when the model tables stay in
    global memory; or dict(refused=True, per_warp) when general_setup refuses the model."""
    ne = model.n_entities
    per_warp = MBAR + warp_block_bytes(model)
    if per_warp > WARP_SMEM_MAX:
        return dict(refused=True, per_warp=per_warp)
    model_bytes = _ceil(ne * A.ENTITY_DTYPE.itemsize + ne * 4 + len(model.backends) * 4, 16)
    if per_warp + model_bytes > WARP_SMEM_MAX:
        model_bytes = 0
    warps = min(8, max(1, (WARP_SMEM_BUDGET // 2) // per_warp))
    while warps > 1 and per_warp * warps + model_bytes > WARP_SMEM_MAX:
        warps -= 1
    smem = per_warp * warps + model_bytes
    ctas_per_sm = max(1, min((227 * 1024) // (smem + 1024), 64 // warps))
    ctas_per_sm = min(ctas_per_sm, 2048 // (warps * 32))
    return dict(refused=False, per_warp=per_warp, model_bytes=model_bytes, warps=warps, smem=smem,
                ctas_per_sm=ctas_per_sm)


def warp_grid(geo, n_replicas, sm_count):
    """launch_warp's grid: one CTA per `warps` replicas, at most ctas_per_sm CTAs per SM (persistent warps)"""
    return min(-(-n_replicas // geo["warps"]), sm_count * geo["ctas_per_sm"])


def fixed_slots(model):
    """launch_thread's entity-owned payload slots: no more entities than future-event slots, no CachingServer, every
    Server at concurrency 1 in every sweep cell, and not a linked partition's destination (no inbox)."""
    if model.n_entities > fel_slots(model, model.inbox_cap) or model.inbox_cap:
        return False
    k, c = model.entities["kind"], model.entities["i0"]
    for i in range(model.n_entities):
        if k[i] == A.HS_ENT_CACHE_SERVER:
            return False
        if k[i] == A.HS_ENT_SERVER:
            cmax = int(c[i]) if model.cell_i0 is None else max(int(c[i]), int(np.asarray(model.cell_i0)[:, i].max()))
            if cmax != 1:
                return False
    return True


# ---- models ------------------------------------------------------------------------------------------------------------

def farm(n_servers, *, rate=None, mean_s=0.1, key_table=None):
    """Source.poisson -> LoadBalancer (round robin, or ``key_table``) -> n concurrency-1 exponential servers -> Sink,
    each server at rho = 0.8 by default."""
    rate = 8.0 * n_servers if rate is None else rate
    if key_table is not None:
        return hs.lb_key_table(key_table, n_servers, rate, mean_service_s=mean_s)
    return hs.lb_round_robin(n_servers, rate, mean_service_s=mean_s)


CONFIGS3_VNODES, CONFIGS3_KEYS = 100, 10000


def configs3_table():
    """BASELINE configs[3]'s key table: 10 000 client ids over the consistent-hash ring of S0..S1023, 100 virtual
    nodes each"""
    return hs.consistent_hash_table([f"S{i}" for i in range(1024)], CONFIGS3_VNODES, CONFIGS3_KEYS)


def sink_fan(n_sinks, rate):
    """Source.poisson -> LoadBalancer (round robin) -> n Sinks: every Sink collects its own latency samples."""
    b = hs.ModelBuilder()
    src = b.source(rate=rate)
    sinks = [b.sink(f"Sink{i}") for i in range(n_sinks)]
    lb = b.load_balancer(backends=sinks)
    b.set_target(src, lb)
    return b.build()


def counter_fan(n_counters, rate, *, probe_on=None):
    """Source.poisson -> LoadBalancer (round robin) -> n Counters; with ``probe_on`` = k a Probe sampling Counter k's
    total every 0.1 s (its two rows come last)."""
    b = hs.ModelBuilder()
    src = b.source(rate=rate)
    counters = [b.counter(f"C{i}") for i in range(n_counters)]
    b.set_target(src, b.load_balancer(backends=counters))
    if probe_on is not None:
        b.probe(target=counters[probe_on], metric="total", interval_s=0.1)
    return b.build()


def wide_server(concurrency, rate, service_s, *, exponential=False):
    """Source.poisson -> one Server(concurrency, constant or exponential service) -> Sink.  A server whose every slot
    is busy holds ``concurrency`` pending continuations."""
    return hs.mm1(rate=rate, mean_service_s=service_s, concurrency=concurrency, exponential=exponential)


SKETCH_KEYS = 4000


def big_sketches(rate=8000.0):
    """Keyed Poisson requests (4 000 keys) through a round-robin LoadBalancer into seven servers, each feeding one sketch
    at the top of its range, and a CachingServer with 2^20 key slots (8 MB of insertion times per replica): HLL p = 16
    from a table and hashed on the device (K = 0), a 2 719 x 7 Count-Min sketch, a Bloom filter of 2^20 + 1 bits, TopK
    k = 512, a TDigest at compression 400 and a reservoir of 5 000."""
    K = SKETCH_KEYS
    b = hs.ModelBuilder()
    src = b.source(rate=rate, key_population=K)
    sketches = [
        b.sketch_hll("hll16_table", precision=16, table=hs.hll_table(16, 3, K)),
        b.sketch_hll("hll16_hashed", precision=16, seed=5),
        b.sketch_cms("cms_2719x7", width=2719, depth=7, table=hs.cms_table(2719, 7, 7, K)),
        b.sketch_bloom("bloom_2p20p1", size_bits=(1 << 20) + 1, num_hashes=5, seed=9),
        b.sketch_topk("topk512", k=512, key_population=K),
        b.sketch_tdigest("tdigest400", compression=400.0),
        b.sketch_reservoir("reservoir5000", size=5000, key_population=K, seed=11),
    ]
    servers = [b.server(f"S{i}", mean_service_s=0.8 * 8 / rate) for i in range(len(sketches))]
    cache = b.cache_server(key_slots=1 << 20, cache_ttl_s=0.05, datastore_read_latency_s=0.002)
    b.set_target(src, b.load_balancer(backends=servers + [cache]))
    for sv, sk in zip(servers, sketches):
        b.set_target(sv, sk)
    return b.build()


# ---- the thread engine's slot and entity limits -----------------------------------------------------------------------
#
# A server with concurrency c holds one pending continuation per busy slot.  A push takes the slot id on top of the
# free-slot stack, which starts sorted, so it is the heap's size while the stack's top has not been used yet: once more
# than 2^15 requests are in service, slot ids above 2^15 are handed out.  The long constant service of the wide server
# pops those only after the horizon, so a second, short server next to it takes them: each of its continuations gets a
# slot id near the heap's size and is popped 10 ms later.
# Two Poisson arrivals on the same nanosecond leave a request in the queue with no poll pending (the reference's
# QueueDriver polls on an empty-to-non-empty enqueue and on a completion only), and from then on the server takes one
# request per completion: a few percent of the replicas stall there, at any fill level.  The rate is low and the
# service long so that most replicas fill before such a collision: 2 000 arrivals/s for 17.5 s.

def slot_server(concurrency=36500, *, rate=2000.0, service_s=17.5, capacity=1024):
    """Source.poisson -> Server(c, constant service) -> Sink, and Source.poisson(50/s) -> Server(1, exponential 10 ms)
    -> the same Sink.  The bounded queues (``capacity``) keep a stalled replica's queue inside a ring of that size."""
    b = hs.ModelBuilder()
    sink = b.sink()
    wide = b.server("Wide", concurrency=concurrency, mean_service_s=service_s, exponential=False, capacity=capacity,
                    downstream=sink)
    short = b.server("Short", mean_service_s=0.01, capacity=capacity, downstream=sink)
    b.source("WideSource", rate=rate, target=wide)
    b.source("ShortSource", rate=50.0, target=short)
    return b.build()


SLOT_END_NS = 18 * 10**9             # slot_server(): about 35 000 requests in service from 17.5 s on
MAX_SLOT_C = 65473                   # S = 24 + 2 x 2 + (c + 1) + 2 = 65 504, the largest S general_setup accepts
MAX_SLOT_END_NS = 33_600_000_000     # slot_server(MAX_SLOT_C, service_s=33.0): every slot busy from about 32.7 s on
N_FAN_COUNTERS = 65531               # counter_fan(N, probe_on=N - 1): 65 535 rows, the most hs_model_validate accepts
FAN_RATE, FAN_END_NS = 80000.0, 10**9


def max_counter_fan():
    return counter_fan(N_FAN_COUNTERS, FAN_RATE, probe_on=N_FAN_COUNTERS - 1)


# ---- reference fixtures (tests/golden/gen_model_size_golden.py -> tests/golden/size_<name>.npz) ------------------------

FIXTURE_SEED = 23
FIXTURE_TAIL = 64                    # records and samples kept from the end of the run


def fixture_models():
    """name -> (model, end_ns, ref_harness.run_reference keywords): the models of the marked rows, short horizons"""
    return {
        "farm512": (farm(512), 300_000_000, {}),
        "farm1024_rr": (farm(1024), 200_000_000, {}),
        "farm1024_configs3": (farm(1024, key_table=configs3_table(), rate=8192.0), 200_000_000,
                              dict(chash_vnodes=CONFIGS3_VNODES)),
        "slot_server": (slot_server(), SLOT_END_NS, {}),
        "counter_fan": (max_counter_fan(), FAN_END_NS, {}),
    }
