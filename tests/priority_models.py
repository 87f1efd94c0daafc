"""Models with PriorityQueue servers: the reference fixtures (tests/golden/gen_priority_golden.py) and seeded random
models that mix priority servers with FIFO / LIFO servers, load balancers, sinks, counters and probes.  Test
infrastructure.

Each builder returns (FlatModel, end_seconds, extras).  extras["priorities"] maps a server's entity id to the values
its PriorityByKey holds exactly as the reference receives them (ints, bools, -0.0 stay what they are; the FlatModel
holds them as doubles), extras["zipf_s"] the Zipf exponent of each Zipf source."""
import numpy as np

import happysim_b200 as hs


class _Builder:
    def __init__(self):
        self.b = hs.ModelBuilder()
        self.extras = {"priorities": {}, "zipf_s": {}}

    def source(self, name, K, *, zipf_s=None, **kw):
        if zipf_s is not None:
            kw["key_cdf"] = hs.zipf_cdf(K, zipf_s)
        i = self.b.source(name, key_population=K, **kw)
        if zipf_s is not None:
            self.extras["zipf_s"][i] = zipf_s
        return i

    def server(self, name, *, values=None, **kw):
        i = self.b.server(name, priorities=None if values is None else [float(v) for v in values], **kw)
        if values is not None:
            self.extras["priorities"][i] = list(values)
        return i


def _finish(B, end_s):
    return B.b.build(), float(end_s), B.extras


def fixture_models():
    """name -> (FlatModel, end_seconds, extras): the models whose reference runs are committed as tests/golden/prio_*.npz."""
    out = {}

    B = _Builder()                                         # M/M/1, two classes: 20 % of the keys priority 0
    src = B.source("Src", 10, rate=9.0)
    srv = B.server("Srv", values=[0, 0] + [1] * 8, mean_service_s=0.1)
    B.b.set_target(src, srv); B.b.set_target(srv, B.b.sink("Sink"))
    out["mm1_two_class"] = _finish(B, 60)

    B = _Builder()                                         # Zipf keys, priority = rank
    src = B.source("Src", 50, zipf_s=1.1, rate=9.0)
    srv = B.server("Srv", values=list(range(50)), mean_service_s=0.1)
    B.b.set_target(src, srv); B.b.set_target(srv, B.b.sink("Sink"))
    out["zipf_rank"] = _finish(B, 60)

    B = _Builder()                                         # a bounded heap that drops
    src = B.source("Src", 4, rate=12.0)
    srv = B.server("Srv", values=[2.0, 1.0, 0.0, 3.0], mean_service_s=0.1, capacity=8)
    B.b.set_target(src, srv); B.b.set_target(srv, B.b.sink("Sink"))
    out["bounded_drops"] = _finish(B, 40)

    B = _Builder()                                         # c = 4
    src = B.source("Src", 6, rate=36.0)
    srv = B.server("Srv", values=[0.25, 3.5, 1.0, 0.25, 2.0, 1.0], mean_service_s=0.1, concurrency=4)
    B.b.set_target(src, srv); B.b.set_target(srv, B.b.sink("Sink"))
    out["c4"] = _finish(B, 30)

    B = _Builder()                                         # RoundRobin onto 8 priority servers
    src = B.source("Src", 8, rate=70.0)
    snk = B.b.sink("Sink")
    servers = []
    for k in range(8):
        servers.append(B.server(f"S{k}", values=[(k + j) % 3 for j in range(8)], mean_service_s=0.1))
        B.b.set_target(servers[-1], snk)
    lb = B.b.load_balancer("LB", backends=servers)
    B.b.set_target(src, lb)
    out["rr8"] = _finish(B, 20)

    B = _Builder()                                         # arrivals and completions tie at one nanosecond, equal priorities
    s1 = B.source("SrcA", 4, rate=10.0, poisson=False)
    s2 = B.source("SrcB", 4, rate=10.0, poisson=False)
    srv = B.server("Srv", values=[1.0, 1.0, 1.0, 0.0], mean_service_s=0.1, exponential=False)
    B.b.set_target(s1, srv); B.b.set_target(s2, srv); B.b.set_target(srv, B.b.sink("Sink"))
    out["tie_insertion_order"] = _finish(B, 12)

    B = _Builder()                                         # negative, -0.0 / 0.0, int and bool priorities
    src = B.source("Src", 7, rate=9.0)
    srv = B.server("Srv", values=[-1.5, -0.0, 0.0, 2, -3, True, 7], mean_service_s=0.1)
    B.b.set_target(src, srv); B.b.set_target(srv, B.b.counter("Counter"))
    out["signs_ints"] = _finish(B, 40)

    B = _Builder()                                         # a Probe on depth (len(heap))
    src = B.source("Src", 10, rate=9.5)
    srv = B.server("Srv", values=[0, 1, 1, 1, 1, 0, 1, 1, 1, 1], mean_service_s=0.1)
    B.b.set_target(src, srv); B.b.set_target(srv, B.b.sink("Sink"))
    B.b.probe("DepthProbe", target=srv, metric="depth", interval_s=0.25)
    out["probe_depth"] = _finish(B, 30)
    return out


RANDOM_SEEDS = list(range(60))


def random_priority_model(seed: int):
    """A seeded random model: one or two keyed sources (uniform or Zipf), a load balancer or a single entry server,
    servers with PriorityQueue / FIFO / LIFO queues (random capacities, concurrency, service distributions, tables of
    ints and floats, negative ones and ties included), tandem hops, sinks, counters and probes."""
    rng = np.random.RandomState(10_000 + seed)
    B = _Builder()
    K = int(rng.choice([2, 5, 16, 40]))
    zs = float(rng.choice([0.7, 1.2])) if rng.rand() < 0.4 else None
    n_src = 1 + int(rng.rand() < 0.35)
    rate = float(rng.choice([15.0, 30.0, 50.0]))

    def table():
        if rng.rand() < 0.5:
            return [int(x) for x in rng.randint(-2, 3, size=K)]
        return [float(x) for x in np.round(rng.uniform(-1.0, 2.0, size=K), 2)]

    def leaf():
        r = rng.rand()
        return B.b.sink(f"Sink{len(B.b._rows)}") if r < 0.7 else B.b.counter(f"Counter{len(B.b._rows)}")

    def server(name, downstream):
        pol = rng.choice(["prio", "prio", "fifo", "lifo"])
        kw = dict(concurrency=int(rng.choice([1, 1, 2, 3])), mean_service_s=float(rng.choice([0.02, 0.05, 0.1])),
                  exponential=bool(rng.rand() < 0.8), capacity=int(rng.choice([-1, -1, 3, 6, 20])))
        i = B.server(name, values=table() if pol == "prio" else None, lifo=(pol == "lifo"), **kw)
        B.b.set_target(i, downstream)
        return i

    n_back = int(rng.choice([1, 1, 3, 5]))
    fronts = []
    for k in range(n_back):
        down = leaf()
        if rng.rand() < 0.3:                               # tandem: a second hop
            down = server(f"T{k}", down)
        fronts.append(server(f"S{k}", down))
    entry = fronts[0] if n_back == 1 else B.b.load_balancer("LB", backends=fronts)
    for s in range(n_src):
        i = B.source(f"Src{s}", K, zipf_s=zs, rate=rate / n_src, poisson=bool(rng.rand() < 0.85))
        B.b.set_target(i, entry)
    if rng.rand() < 0.4:
        B.b.probe("Probe", target=fronts[int(rng.randint(n_back))], metric=str(rng.choice(["depth", "stats_accepted", "active_requests"])),
                  interval_s=float(rng.choice([0.1, 0.3])))
    return _finish(B, float(rng.choice([4.0, 8.0])))
