"""Seeded random models over everything the lowering supports (sources with rate profiles, stop times and
uniform / Zipf client ids; load balancers; tandem, bounded, LIFO and multi-slot servers; sinks, counters, probes
and the five sketch collectors).  Test infrastructure: the differential tests run each model on the CPU oracle
and on the device engines and compare every output bit for bit."""
import numpy as np

import happysim_b200 as hs
from happysim_b200 import _abi as A


def random_model(seed: int, with_extras: bool = False):
    """-> (FlatModel, end_seconds, description[, extras for tests/golden/ref_harness.run_reference])"""
    rng = np.random.RandomState(seed)
    extras = {"zipf_s": {}, "sketch_seeds": {}, "random_key_table": False}
    b = hs.ModelBuilder()
    K = int(rng.choice([0, 0, 16, 200]))
    zipf = K > 0 and rng.rand() < 0.5
    n_src = 1 + int(rng.rand() < 0.3)
    base_rate = float(rng.choice([20.0, 60.0, 120.0]))
    srcs = []
    for i in range(n_src):
        kw = dict(rate=base_rate / n_src, poisson=bool(rng.rand() < 0.7), key_population=K)
        if rng.rand() < 0.2:
            kw["stop_after_ns"] = int(rng.uniform(0.5, 3.0) * 1e9)
        r = rng.rand()
        if r < 0.15:
            kw["profile"] = ("linear_ramp", float(rng.uniform(1, 4)), kw["rate"], kw["rate"] * float(rng.uniform(0.5, 2.0)))
        elif r < 0.3:
            kw["profile"] = ("spike", kw["rate"], kw["rate"] * 3.0, float(rng.uniform(0.2, 1.5)), float(rng.uniform(0.2, 1.0)))
        zs = float(rng.choice([0.0, 0.8, 1.3]))
        if zipf:
            kw["key_cdf"] = hs.zipf_cdf(K, zs)
        srcs.append(b.source(f"Src{i}", **kw))
        if zipf:
            extras["zipf_s"][srcs[-1]] = zs

    def sink():
        kinds = ["sink", "counter", "tdigest"] + (["hll", "cms", "bloom", "topk"] if K else [])
        k = kinds[rng.randint(len(kinds))]
        if k == "sink":
            return b.sink(f"Sink{b_count()}")
        if k == "counter":
            return b.counter(f"Counter{b_count()}")
        if k == "tdigest":
            return b.sketch_tdigest(f"TD{b_count()}", compression=float(rng.choice([5.0, 20.0])))
        if k == "hll":
            p = int(rng.choice([4, 7]))
            i = b.sketch_hll(f"HLL{b_count()}", precision=p, table=hs.hll_table(p, seed, K))
            extras["sketch_seeds"][i] = seed
            return i
        if k == "cms":
            i = b.sketch_cms(f"CMS{b_count()}", width=9, depth=3, table=hs.cms_table(9, 3, seed, K))
            extras["sketch_seeds"][i] = seed
            return i
        if k == "bloom":
            i = b.sketch_bloom(f"BF{b_count()}", size_bits=77, num_hashes=3, table=hs.bloom_table(77, 3, seed, K))
            extras["sketch_seeds"][i] = seed
            return i
        return b.sketch_topk(f"Top{b_count()}", k=int(rng.choice([2, 6])), key_population=K)

    def b_count():
        return len(b._rows)

    def server(downstream, mean_scale=1.0):
        c = int(rng.choice([1, 1, 2, 4]))
        mean = mean_scale * c / base_rate * float(rng.uniform(0.3, 1.1))
        return b.server(f"Srv{b_count()}", concurrency=c, mean_service_s=mean, exponential=bool(rng.rand() < 0.7),
                        downstream=downstream, capacity=int(rng.choice([-1, -1, -1, 0, 3])), lifo=bool(rng.rand() < 0.3))

    shape = rng.choice(["single", "tandem", "lb", "lb_tandem", "direct"])
    if shape == "direct":
        head = sink()
    elif shape == "single":
        head = server(sink())
    elif shape == "tandem":
        head = server(server(sink()))
    else:
        n = int(rng.randint(2, 6))
        shared = sink() if rng.rand() < 0.5 else None
        backs = []
        for _ in range(n):
            dst = shared if shared is not None else sink()
            if shape == "lb_tandem" and rng.rand() < 0.5:
                dst = server(dst)
            backs.append(server(dst, mean_scale=n))
        table = None
        if K and rng.rand() < 0.6:
            table = rng.randint(0, n, size=K).astype(np.int32)
            extras["random_key_table"] = True
        head = b.load_balancer(f"LB{b_count()}", backends=backs, key_table=table)
    for s in srcs:
        b.set_target(s, head)
    servers = [i for i, r in enumerate(b._rows) if r[0] == hs._abi.HS_ENT_SERVER]
    if servers and rng.rand() < 0.4:
        b.probe("Probe", target=int(rng.choice(servers)), metric=str(rng.choice(["depth", "active_requests", "stats_accepted"])),
                interval_s=float(rng.choice([0.05, 0.25])))
    model = b.build()
    end_s = float(rng.uniform(1.5, 4.0))
    what = f"seed {seed}: {shape}, K={K}{' zipf' if zipf else ''}, {n_src} source(s), {model.n_entities} entities"
    return (model, end_s, what, extras) if with_extras else (model, end_s, what)


def random_lane_model(seed: int):
    """Source -> Server -> Sink | Counter | nothing: the topology the lane engine keeps in registers, with random
    arrival / service kinds, concurrency, queue policy and capacity, stop times and rate profiles.  Constant
    arrivals against constant service times make arrivals and completions collide on the same nanosecond (the
    generic tie path).  -> (FlatModel, end_seconds, description)"""
    rng = np.random.RandomState(10_000 + seed)
    b = hs.ModelBuilder()
    rate = float(rng.choice([4.0, 10.0, 25.0, 100.0]))
    poisson = bool(rng.rand() < 0.6)
    kw = dict(rate=rate, poisson=poisson)
    if rng.rand() < 0.2:
        kw["stop_after_ns"] = int(rng.uniform(0.3, 2.0) * 1e9)
    r = rng.rand()
    if r < 0.12:
        kw["profile"] = ("linear_ramp", float(rng.uniform(1, 3)), rate, rate * float(rng.uniform(0.5, 2.0)))
    elif r < 0.24:
        kw["profile"] = ("spike", rate, rate * 2.5, float(rng.uniform(0.2, 1.0)), float(rng.uniform(0.2, 1.0)))
    src = b.source(**kw)
    c = int(rng.choice([1, 1, 2, 3, 8]))
    exponential = bool(rng.rand() < 0.6)
    # constant/constant with an integer ratio -> exact ties between ticks and completions
    mean = (c / rate) * float(rng.choice([0.5, 1.0, 2.0])) if not exponential and not poisson else (c / rate) * float(rng.uniform(0.3, 1.2))
    srv = b.server(concurrency=c, mean_service_s=mean, exponential=exponential, capacity=int(rng.choice([-1, -1, 0, 2, 5])),
                   lifo=bool(rng.rand() < 0.3))
    dst = int(rng.choice([0, 0, 1, 2]))
    b.set_target(src, srv)
    if dst == 0:
        b.set_target(srv, b.sink())
    elif dst == 1:
        b.set_target(srv, b.counter())
    model = b.build()
    end_s = float(rng.uniform(1.0, 5.0))
    what = (f"lane seed {seed}: rate {rate} {'poisson' if poisson else 'constant'}, c={c}, "
            f"{'exp' if exponential else 'const'} service {mean:.4f}, dst {('sink', 'counter', 'none')[dst]}")
    return model, end_s, what


def random_model_v2(seed: int, with_extras: bool = False):
    """Second generator (round 2 features; its own fixture file so that the first generator's models stay as they
    are): user-defined STEP rate profiles and CachingServer farms behind round-robin / consistent-hash load balancers,
    alone and mixed with ordinary servers.  -> (FlatModel, end_seconds, description[, extras for the harness])"""
    rng = np.random.RandomState(50_000 + seed)
    extras = {"profile_objects": {}, "chash_vnodes": None}
    b = hs.ModelBuilder()
    shape = str(rng.choice(["cache_direct", "cache_lb_rr", "cache_lb_chash", "step_server", "step_farm", "step_cache"]))
    K = int(rng.choice([3, 12, 40])) if "cache" in shape else int(rng.choice([0, 16]))
    rate = float(rng.choice([30.0, 90.0, 200.0]))
    kw = dict(rate=rate, poisson=bool(rng.rand() < 0.75), key_population=K)
    if rng.rand() < 0.15:
        kw["stop_after_ns"] = int(rng.uniform(0.5, 2.0) * 1e9)
    step = None
    if shape.startswith("step") or rng.rand() < 0.3:
        n = int(rng.randint(1, 6))
        breaks = sorted({round(float(x), 3) for x in rng.uniform(0.05, 3.5, size=n)})
        rates = [rate * float(rng.choice([0.3, 0.6, 1.0, 1.7, 2.5])) for _ in range(len(breaks) + 1)]
        step = hs.StepProfile(tuple(breaks), tuple(rates))
        kw["profile"] = ("step", list(step.breakpoints), list(step.rates))
    src = b.source("Src", **kw)
    if step is not None:
        extras["profile_objects"][src] = step

    def cache(i):
        ttl = float(rng.choice([0.05, 0.3, 1.0, 30.0]))
        return b.cache_server(f"Cache{i}", key_slots=K, cache_ttl_s=ttl,
                              cache_read_latency_s=float(rng.choice([0.0001, 0.001])),
                              datastore_read_latency_s=float(rng.choice([0.005, 0.02])),
                              processing_latency_s=float(rng.choice([0.001, 0.004])))

    if shape in ("cache_direct", "step_cache"):
        head = cache(0)
    elif shape == "step_server":
        snk = b.sink()
        c = int(rng.choice([1, 2]))
        head = b.server("Srv", concurrency=c, mean_service_s=c / rate * float(rng.uniform(0.4, 1.0)),
                        exponential=bool(rng.rand() < 0.7), downstream=snk, lifo=bool(rng.rand() < 0.3))
    else:
        n = int(rng.randint(2, 6))
        if shape == "step_farm":
            snk = b.sink()
            backs = [b.server(f"Srv{i}", mean_service_s=n / rate * float(rng.uniform(0.4, 1.0)), downstream=snk) for i in range(n)]
            names = None
        else:
            backs = [cache(i) for i in range(n)]
            names = [f"Cache{i}" for i in range(n)]
        table = None
        if shape == "cache_lb_chash":
            extras["chash_vnodes"] = int(rng.choice([5, 30]))
            table = hs.consistent_hash_table(names, extras["chash_vnodes"], K)
        head = b.load_balancer("LB", backends=backs, key_table=table)
    b.set_target(src, head)
    model = b.build()
    end_s = float(rng.uniform(1.5, 4.0))
    what = f"v2 seed {seed}: {shape}, K={K}, rate {rate}{' step' if step is not None else ''}, {model.n_entities} entities"
    return (model, end_s, what, extras) if with_extras else (model, end_s, what)


FAULT_SEED_OFFSET, FAULT_SEED_OFFSET_V2 = 1000, 5000


def random_fault_plan(model, end_s: float, seed: int, offset: int = FAULT_SEED_OFFSET):
    """A random node-fault schedule for ``model``: 1 to 4 faults (crash, crash with restart, pause) on entities other
    than probes and their tick sources, at times in [0, end_s] rounded to the millisecond, each cancelled with
    probability 0.2.  -> (plan: [(kind, entity name, a_s, b_s)], indices of the cancelled faults)"""
    import random
    rng = random.Random(offset + seed)
    ents = model.entities
    names = [n for i, n in enumerate(model.names) if int(ents["kind"][i]) != A.HS_ENT_PROBE and not (
        int(ents["kind"][i]) == A.HS_ENT_SOURCE and int(ents["kind"][int(ents["target"][i])]) == A.HS_ENT_PROBE)]
    plan = []
    for _ in range(rng.randint(1, 4)):
        nm = rng.choice(names)
        a = round(rng.uniform(0.0, end_s), 3)
        kind = rng.choice(["crash", "crash_restart", "pause"])
        b = round(a + rng.uniform(0.01, end_s / 2), 3)
        plan.append((kind, nm, a, b))
    cancel = [k for k in range(len(plan)) if rng.random() < 0.2]
    return plan, cancel


def _fault_seeds_v1(n=60):
    """the first n seeds of random_model whose model the reference harness can build (no random key table)"""
    out, s = [], 0
    while len(out) < n:
        if not random_model(s, with_extras=True)[3]["random_key_table"]:
            out.append(s)
        s += 1
    return out


FAULT_SEEDS_V1 = _fault_seeds_v1()          # against the reference (CPU) and tests/golden/random_fault_models.npz
FAULT_SEEDS_V2 = list(range(60))


def random_fault_case(version: int, seed: int, scale: float = 1.0):
    """A seeded random model (random_model or random_model_v2) with its random fault plan, drawn on the model's
    horizon times ``scale`` (a shorter run keeps its faults).
    -> (FlatModel without FAULT rows, end_seconds, plan, cancel, run seed, description, extras for the harness)"""
    if version == 1:
        model, end_s, what, ex = random_model(seed, with_extras=True)
        end_s = min(float(end_s), 6.0) * scale
        plan, cancel = random_fault_plan(model, end_s, seed)
        return model, end_s, plan, cancel, seed, what, ex
    model, end_s, what, ex = random_model_v2(seed, with_extras=True)
    end_s = float(end_s) * scale
    plan, cancel = random_fault_plan(model, end_s, seed, FAULT_SEED_OFFSET_V2)
    return model, end_s, plan, cancel, 2000 + seed, what, ex


def fault_schedule(plan, F):
    """``plan`` as a FaultSchedule of the module ``F`` (the reference's happysimulator.faults or the mirror's api)"""
    s = F.FaultSchedule()
    for kind, nm, a, b in plan:
        s.add(F.CrashNode(nm, at=a) if kind == "crash" else F.CrashNode(nm, at=a, restart_at=b) if kind == "crash_restart"
              else F.PauseNode(nm, start=a, end=b))
    return s


def with_faults(model, plan, cancel):
    """``model`` plus one FAULT row per fault event of ``plan``, as lowering.fault_events lowers a FaultSchedule built
    when the Simulation is: a crash (or pause) event and, for crash_restart and pause, a restart (resume) event, at
    Instant.from_seconds of the plan's times; bootstrap sort indices after the sources' and probes' first ticks (one
    SOURCE row each), one per event in schedule order.  Names resolve as FaultSchedule._build_context does, the last of
    the entities, then the sources, winning."""
    import dataclasses
    ents = model.entities
    kinds = ents["kind"]
    order = [i for i in range(model.n_entities) if int(kinds[i]) not in (A.HS_ENT_SOURCE, A.HS_ENT_PROBE, A.HS_ENT_REMOTE)] \
        + [i for i in range(model.n_entities) if int(kinds[i]) == A.HS_ENT_SOURCE]
    by_name = {model.names[i]: i for i in order}
    idx = int((kinds == A.HS_ENT_SOURCE).sum())
    fb = hs.ModelBuilder()
    for k, (kind, nm, a, b) in enumerate(plan):
        for t_s, crash in [(a, True)] + ([] if kind == "crash" else [(b, False)]):
            fb.fault(f"fault:{nm}", target=by_name[nm], time_ns=int(t_s * 1_000_000_000), crash=crash, sort_index=idx,
                     cancelled=k in cancel)
            idx += 1
    return dataclasses.replace(model, entities=np.concatenate([ents, np.array(fb._rows, dtype=A.ENTITY_DTYPE)]),
                               names=list(model.names) + fb._names)


def random_linked_model(seed: int):
    """Random ParallelSimulation with PartitionLinks (SURVEY 8(f) row 4): 2-4 partitions, each an optional source, an
    entry (a server, a two-server chain or a load balancer over two servers), a sink and a counter; the last server of a
    partition forwards to its own sink / counter / key sketch, to the entry of a LATER partition, or back into an EARLIER
    partition's sink or counter.  Links: constant or exponential latency between 1x and 3x the window (exponential:
    plenty of time travel), some lossy, some sharing one latency object.  About a third of the seeds put everything on
    a grid (constant sources, service times and latencies) so that cross-partition events tie with local ones on the
    nanosecond.  -> (LinkedModel, end_seconds, description)"""
    from happysim_b200.linked import LinkedModel, LinkSpec
    rng = np.random.RandomState(70_000 + seed)
    nP = int(rng.randint(2, 5))
    W = float(rng.choice([0.02, 0.05, 0.1]))
    grid = bool(rng.rand() < 0.35)
    K = int(rng.choice([0, 0, 20]))
    builders, info = [], []
    for p in range(nP):
        b = hs.ModelBuilder()
        ids = {}
        has_src = p == 0 or rng.rand() < 0.55
        rate = float(rng.choice([50.0, 100.0])) if grid else float(rng.choice([20.0, 60.0, 150.0]))
        if has_src:
            ids["src"] = b.source(f"P{p}.src", rate=rate, poisson=(not grid) and bool(rng.rand() < 0.75), key_population=K)

        def server(name, n_par=1):
            c = int(rng.choice([1, 1, 2, 3]))
            if grid:
                svc, expo = float(rng.choice([0.005, 0.01])), False
            else:
                svc, expo = c * n_par / (rate * 1.6) * float(rng.uniform(0.5, 1.1)), bool(rng.rand() < 0.7)
            return b.server(name, concurrency=c, mean_service_s=svc, exponential=expo,
                            capacity=int(rng.choice([-1, -1, 2, 6])), lifo=bool(rng.rand() < 0.25))
        shape = str(rng.choice(["one", "chain", "lb"]))
        if shape == "one":
            tail = [server(f"P{p}.s0")]
            ids["entry"] = tail[0]
        elif shape == "chain":
            s0, s1 = server(f"P{p}.s0"), server(f"P{p}.s1")
            b.set_target(s0, s1)
            ids["entry"], tail = s0, [s1]
        else:
            tail = [server(f"P{p}.s0", 2), server(f"P{p}.s1", 2)]
            ids["entry"] = b.load_balancer(f"P{p}.lb", backends=tail)
        ids["sink"], ids["counter"] = b.sink(f"P{p}.sink"), b.counter(f"P{p}.counter")
        if K:
            ids["sketch"] = b.sketch_topk(f"P{p}.heavy", k=5, key_population=K)
        if has_src:
            b.set_target(ids["src"], ids["entry"])
        builders.append(b)
        info.append((ids, tail))
    links: list[list] = [[] for _ in range(nP)]
    shared = {}
    rems = {}
    any_link = False
    for p in range(nP):
        ids, tail = info[p]
        for k, sv in enumerate(tail):
            must = (p == 0 and k == 0 and not any_link)
            choice = "fwd" if must else str(rng.choice(["sink", "counter", "sketch", "fwd", "fwd", "back"]))
            if choice == "sketch" and not K:
                choice = "sink"
            if choice == "fwd" and p == nP - 1:
                choice = "back"
            if choice == "back" and p == 0:
                choice = "counter"
            if choice in ("sink", "counter", "sketch"):
                builders[p].set_target(sv, ids[choice])
                continue
            q = int(rng.randint(p + 1, nP)) if choice == "fwd" else int(rng.randint(0, p))
            dest = info[q][0]["entry"] if choice == "fwd" else info[q][0][str(rng.choice(["sink", "counter"]))]
            slot = next((s for s, l in enumerate(links[p]) if l.dest == q), None)
            if slot is None:
                if grid:
                    kind, mean = A.HS_SVC_CONSTANT, W * float(rng.choice([1.0, 2.0]))
                else:
                    kind = A.HS_SVC_EXPONENTIAL if rng.rand() < 0.4 else A.HS_SVC_CONSTANT
                    mean = W * float(rng.choice([1.0, 1.5, 3.0]))
                stream = shared.setdefault((kind, mean), len(shared))
                slot = len(links[p])
                links[p].append(LinkSpec(q, kind, mean, float(rng.choice([0.0, 0.0, 0.1, 0.3])) if not grid else 0.0, stream))
            rem = rems.get((p, q, dest))          # one REMOTE row per remote entity, as the lowering produces them
            if rem is None:
                rem = rems[(p, q, dest)] = builders[p].remote(f"P{q}.{dest}@P{p}", link=slot, dest_entity=dest)
            builders[p].set_target(sv, rem)
            any_link = True
    models = [b.build() for b in builders]
    for p, m in enumerate(models):
        m.outbox_cap = 256 if m.ids_of(A.HS_ENT_REMOTE) else 0
        m.inbox_cap = 256 if any(l.dest == p for ls in links for l in ls) else 0
    lm = LinkedModel(models, [f"P{p}" for p in range(nP)], links, window_s=W, n_streams=max(1, len(shared)))
    lm.validate()
    end_s = round(float(rng.uniform(1.0, 2.5)), 2)
    while True:          # an end time that does not survive ns -> float seconds -> ns sends the reference's coordinator into
        try:             # an endless loop (the clamped last window ends 1 ns short, coordinator.py:88-95): not a test case
            lm.window_ends(int(end_s * 1e9))
            break
        except ValueError:
            end_s = round(end_s + 0.01, 2)
    what = f"linked seed {seed}: {nP} partitions, window {W}, {'grid' if grid else 'continuous'}, K={K}, " \
           f"{sum(len(l) for l in links)} links, {sum(m.n_entities for m in models)} entities"
    return lm, end_s, what


LINKED_SEEDS = 72
