"""Sweep cells on any lowered model.  A cell is one configuration of a sweep run inside a shared launch: the model's
``cell_d0`` / ``cell_i0`` give every row its d0 (rate, mean service time, TTL, compression) and every SERVER row its i0
(concurrency), and replica g runs cell (g / replicas_per_cell) % n_cells.  ``with_cells`` draws cells that vary every
column api._same_topology lets vary; ``cell_model`` is the plain model of one cell, the single run a cell must equal.
Test infrastructure."""
import dataclasses

import numpy as np

import happysim_b200 as hs
from happysim_b200 import _abi as A
from random_models import random_fault_case, random_lane_model, random_model, random_model_v2, with_faults

TTLS = (0.05, 0.3, 1.0, 30.0)          # seconds: at 12 to 40 keys and 30 to 200 req/s these move keys between hit and miss
TDIGEST_STEPS = (0.0, 0.1, 0.2, 0.45)  # compression offsets that keep the buffer size int(2c)


def with_cells(model, rng, n_cells: int, concurrency: str | None = None):
    """A copy of ``model`` with ``n_cells`` cells; cell 0 is the copy's own rows.  The other cells scale the rate of
    every source without a profile by 0.5 to 1.5, give every server a concurrency from {1, 2, 3, 4} and a mean service
    time scaled with it, every CachingServer a TTL from TTLS and every TDigest a compression of the same int(2c).
    ``concurrency``: "one" (every server of every cell, cell 0 included, at c = 1), "mixed" (c = 1 and c > 1 both
    among the cells of every server) or "any"; None draws one of the three."""
    if concurrency is None:
        concurrency = str(rng.choice(["one", "mixed", "any"]))
    if concurrency == "mixed" and n_cells < 3:
        raise ValueError("mixed concurrency needs at least three cells")
    E = model.entities.copy()
    kind = E["kind"]
    srv = np.flatnonzero(kind == A.HS_ENT_SERVER)
    if concurrency == "one":
        E["d0"][srv] = E["d0"][srv] / np.maximum(E["i0"][srv], 1)
        E["i0"][srv] = 1
    cd = np.tile(E["d0"].astype(np.float64), (n_cells, 1))
    ci = np.tile(E["i0"].astype(np.int32), (n_cells, 1))
    for c in range(1, n_cells):
        for i in range(len(E)):
            k = int(kind[i])
            if k == A.HS_ENT_SOURCE and int(E["i3"][i]) == 0:
                cd[c, i] = E["d0"][i] * float(rng.uniform(0.5, 1.5))
            elif k == A.HS_ENT_SERVER:
                c0 = int(E["i0"][i])
                if concurrency == "one":
                    cv = 1
                elif concurrency == "mixed":
                    cv = 1 if c % 2 == 1 else int(rng.choice([2, 3, 4]))
                else:
                    cv = int(rng.choice([1, 2, 3, 4]))
                ci[c, i] = cv
                cd[c, i] = E["d0"][i] * cv / c0 * float(rng.uniform(0.6, 1.2))
            elif k == A.HS_ENT_CACHE_SERVER:
                cd[c, i] = float(rng.choice(TTLS))
            elif k == A.HS_ENT_SKETCH and int(E["i0"][i]) == A.HS_SK_TDIGEST:
                cd[c, i] = int(E["i2"][i]) / 2.0 + float(rng.choice(TDIGEST_STEPS))
    return dataclasses.replace(model, entities=E, cell_d0=cd, cell_i0=ci)


def cell_model(model, c: int):
    """The plain model (no cells) with cell ``c``'s d0 and i0 written into its rows."""
    E = model.entities.copy()
    E["d0"] = model.cell_d0[c]
    E["i0"] = model.cell_i0[c]
    return dataclasses.replace(model, entities=E, cell_d0=None, cell_i0=None)


def cells_of(n_replicas: int, n_cells: int, replica_index_base: int = 0, replicas_per_cell: int = 1):
    """the cell of every replica of a launch"""
    return ((replica_index_base + np.arange(n_replicas)) // replicas_per_cell) % n_cells


# ---- the sources: the seeded random generators ------------------------------------------------------------------------

def _case_rng(version, seed):
    return np.random.RandomState(90_000 + 1000 * version + seed)


def cell_case(version: str, seed: int, n_cells: int | None = None, concurrency: str | None = None):
    """A random model with cells.  ``version``: "v1" (random_model), "v2" (random_model_v2: step profiles and CachingServer
    farms), "fault" (random_model with its random fault plan) or "lane" (random_lane_model).
    -> (model with cells, end_ns, run seed, description)"""
    rng = _case_rng({"v1": 1, "v2": 2, "fault": 3, "lane": 4}[version], seed)
    n = int(rng.randint(3, 6)) if n_cells is None else n_cells
    if version == "v1":
        m, end_s, what = random_model(seed)
        run_seed = 1000 + seed
    elif version == "v2":
        m, end_s, what = random_model_v2(seed)
        run_seed = 2000 + seed
    elif version == "fault":
        m, end_s, plan, cancel, run_seed, what, _ = random_fault_case(1, seed)
        m = with_faults(m, plan, cancel)
    else:
        m, end_s, what = random_lane_model(seed)
        run_seed = 77 + seed
    cm = with_cells(m, rng, n, concurrency)
    return cm, int(end_s * 1e9), run_seed, f"{what}; {n} cells"


def has_kind(model, kind) -> bool:
    return bool((model.entities["kind"] == kind).any())


def has_tdigest(model) -> bool:
    E = model.entities
    return bool(((E["kind"] == A.HS_ENT_SKETCH) & (E["i0"] == A.HS_SK_TDIGEST)).any())


# ---- the reference fixture's models (tests/golden/sweep_cells.npz) --------------------------------------------------------

FIXTURE_SEED, FIXTURE_END_NS = 31, 3 * 10**9
CACHE_TTLS = (0.05, 0.3, 1.0, 30.0)
TDIGEST_COMPRESSIONS = (20.0, 20.2, 20.45)


def cache_farm(ttl: float = CACHE_TTLS[0]):
    """200 req/s over 12 keys, round robin over three CachingServers"""
    b = hs.ModelBuilder()
    src = b.source("Src", rate=200.0, key_population=12)
    caches = [b.cache_server(f"Cache{i}", key_slots=12, cache_ttl_s=ttl, cache_read_latency_s=0.001,
                             datastore_read_latency_s=0.02, processing_latency_s=0.004) for i in range(3)]
    b.set_target(src, b.load_balancer("LB", backends=caches))
    return b.build()


def tdigest_farm(compression: float = TDIGEST_COMPRESSIONS[0]):
    """120 req/s round robin over four exponential servers into one QuantileEstimator"""
    b = hs.ModelBuilder()
    src = b.source("Src", rate=120.0)
    td = b.sketch_tdigest("Latency", compression=compression)
    servers = [b.server(f"Srv{i}", mean_service_s=0.025, downstream=td) for i in range(4)]
    b.set_target(src, b.load_balancer("LB", backends=servers))
    return b.build()


def fixture_models():
    """name -> (model with one cell per configuration, [plain model of each configuration])"""
    out = {}
    for name, mk, vals in (("cache_ttl", cache_farm, CACHE_TTLS), ("tdigest_compression", tdigest_farm, TDIGEST_COMPRESSIONS)):
        plains = [mk(v) for v in vals]
        m = dataclasses.replace(plains[0], cell_d0=np.stack([p.entities["d0"].astype(np.float64) for p in plains]),
                                cell_i0=np.stack([p.entities["i0"].astype(np.int32) for p in plains]))
        out[name] = (m, plains)
    return out
