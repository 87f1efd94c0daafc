"""SURVEY 8(f) row 3 on the CPU side: sketch state layout, the host hash tables and the mirror classes
against the answers the reference's own HyperLogLog / CountMinSketch gave (tests/golden/philox_sketch_*),
merge contracts, lowering and validation."""
import ctypes as C

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A, distributed as D, engine, lowering, results
from happysim_b200.engine import EngineError


def farm_model():
    m, kw, z = G.load("philox_sketch_cms_farm")
    return m, kw, z


def test_layout_matches_the_c_rule_in_both_libraries():
    m, _, _ = farm_model()
    per, mer, total, mtotal = m.sketch_layout()
    for L in (O.lib(), engine.load_library()):
        n = m.n_entities
        a, b = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        t, mt = C.c_uint64(), C.c_uint64()
        d = m.desc()
        assert L.hs_sketch_layout(C.byref(d), a, b, C.byref(t), C.byref(mt)) == 0
        assert list(a) == per and list(b) == mer and t.value == total and mt.value == mtotal
    assert total == 3 * 16 * 4 + 16 and mtotal == (3 * 16 * 8) + 16        # CMS 3x16, HLL p=4


@pytest.mark.parametrize("name", G.case_names("philox_sketch_"))
def test_mirror_classes_give_the_reference_answers(name):
    """Oracle state == reference state (test_oracle_golden); here: our cardinality() / estimate() computed from
    that state == the reference objects' answers, and the host tables == the reference's hashing."""
    m, kw, z = G.load(name)
    out = O.oracle_run(m, O.make_params(n_replicas=1, **G.caps(z), **kw))
    G.check_against(z, out)
    views = m.sketch_views(out["sketches"])
    for i, state in views.items():
        e = m.entities[i]
        seed = int(z[f"sketch_seed_{i}"]) if f"sketch_seed_{i}" in z.files else -1     # TopK takes no seed
        seed = None if seed < 0 else seed
        want = z[f"sketch_answer_{i}"]
        added = int(out["entity_stats"][0][i]["c1"])
        if int(e["i0"]) == A.HS_SK_HLL:
            sk = hs.HyperLogLog(precision=int(e["i2"]), seed=seed)
            sk._load_device_state(state[0], added)
            assert sk.cardinality() == int(want[0]) and sk.item_count == added
        elif int(e["i0"]) == A.HS_SK_BLOOM:
            sk = hs.BloomFilter(size_bits=int(e["i3"]), num_hashes=int(e["i2"]), seed=seed)
            sk._load_device_state(state[0], added)
            K = int(e["l0"])
            assert [int(sk.contains(k)) for k in range(K)] == [int(x) for x in want[:K]]
            assert sk._bits_set == int(want[K]) and sk.item_count == added and 0 < sk.fill_ratio < 1
        elif int(e["i0"]) == A.HS_SK_TDIGEST:
            sk = hs.TDigest(compression=float(e["d0"]))
            sk._load_device_state(state[0])
            assert sk.item_count == added and len(sk._buffer) > 0          # state as left by add(): unflushed values
            qs = [0.0, 0.001, 0.01, 0.25, 0.5, 0.75, 0.9, 0.99, 0.999, 1.0]
            vals = [sk.quantile(q) for q in qs] + [sk.cdf(v) for v in (0.0, 0.01, 0.05, 0.1, 0.3, 1.0, 5.0)] + \
                   [float(sk.centroid_count)]
            assert np.array(vals, dtype=np.float64).view(np.int64).tolist() == [int(x) for x in want]   # bit for bit
            assert sk.percentile(50) == sk.quantile(0.5) and sk.min <= sk.quantile(0.5) <= sk.max
        elif int(e["i0"]) == A.HS_SK_RESERVOIR:
            sk = hs.ReservoirSampler(size=int(e["i2"]))
            untouched = sk._rng.getstate()
            sk._load_device_state(state[0], added)
            assert sk.sample() == [int(x) for x in want[:-2]] and sk.item_count == added == int(want[-2])
            assert len(sk) == min(added, sk.capacity) and sk.is_full == (added >= sk.capacity)
            if added:                       # the generator continues where the reference's own would
                assert sk._rng.getrandbits(32) == int(want[-1])
            else:
                assert sk._rng.getstate() == untouched
        elif int(e["i0"]) == A.HS_SK_TOPK:
            sk = hs.TopK(k=int(e["i2"]))
            sk._load_device_state(state[0], added)
            flat = [v for fe in sk.top() for v in (fe.item, fe.count, fe.error)] + [sk.max_error(), sk.guaranteed_threshold()]
            assert flat == [int(x) for x in want]
            assert sk.tracked_count == min(int(e["i2"]), sk.tracked_count) and sk.item_count == added
        else:
            sk = hs.CountMinSketch(width=int(e["i3"]), depth=int(e["i2"]), seed=seed)
            sk._load_device_state(state[0], added)
            assert [sk.estimate(k) for k in range(int(e["l0"]))] == [int(x) for x in want]
            assert int(state[0].sum()) == added * int(e["i2"])           # every add touches one cell per row


def test_tdigest_host_mirror_equals_the_shared_c_step_and_merges():
    """TDigest.add on the host vs csrc/hs_sketch.h through the oracle on the same latency stream (a Sink in
    parallel records it), over many flush/compress rounds; then the order-dependent merge over replicas."""
    b = hs.ModelBuilder()
    src = b.source(rate=400.0)
    s1 = b.server("A", concurrency=4, mean_service_s=0.005, downstream=-1)
    q = b.sketch_tdigest("lat", compression=30.0)
    b.set_target(src, s1); b.set_target(s1, q)
    m = b.build()
    m2 = hs.mm1(rate=400.0, mean_service_s=0.005, concurrency=4)           # same ids: Source, Server, then the sink
    p = dict(seed=7, end_ns=3 * 10**9, n_replicas=3)
    out = O.oracle_run(m, O.make_params(**p))
    ref = O.oracle_run(m2, O.make_params(sample_cap=4000, **p))
    digests = []
    for r in range(3):
        n = int(ref["summaries"][r]["n_sink_samples"])
        mirror = hs.TDigest(30.0)
        for v in ref["sink_samples"][r][:n]["latency_s"]:
            mirror.add(float(v))
        dev = hs.TDigest(30.0); dev._load_device_state(m.sketch_views(out["sketches"])[q][r])
        assert n > 1000 and dev.item_count == n == int(out["entity_stats"][r][q]["c1"])
        assert (dev._means, dev._counts, dev._buffer) == (mirror._means, mirror._counts, mirror._buffer)
        assert (dev.min, dev.max) == (mirror.min, mirror.max) and dev.quantile(0.99) == mirror.quantile(0.99)
        digests.append(dev)
    merged = D.merge_sketch_states(m, out["sketches"])[q]
    acc = hs.TDigest(30.0)
    for d in digests:
        acc.merge(d)
    assert merged._means == acc._means and merged._counts == acc._counts and merged.item_count == sum(d.item_count for d in digests)
    assert acc.quantile(0.5) > 0 and acc.cdf(acc.quantile(0.5)) == pytest.approx(0.5, abs=0.05)


def test_space_saving_host_mirror_equals_the_shared_c_step():
    """TopK.add on the host (dict order) vs csrc/hs_sketch.h's slot array, through the oracle: a direct
    Source -> TopK model sees the raw key stream, which is replayed into the mirror."""
    K, k = 25, 6
    b = hs.ModelBuilder()
    src = b.source(rate=400.0, key_population=K)
    top = b.sketch_topk("heavy", k=k, key_population=K)
    b.set_target(src, top)
    m = b.build()
    p = dict(seed=5, end_ns=10**9, n_replicas=3)
    out = O.oracle_run(m, O.make_params(**p))
    for r in range(3):
        mirror = hs.TopK(k)
        n = int(out["entity_stats"][r][top]["c1"])
        for d in range(n):      # the source's routing draws (hs_handlers.inc / oracle: int(u * K))
            u = O.lib().hs_cpu_uniform(5, r, A.HS_STREAM_ROUTING | (src << 8), d)
            mirror.add(int(u * K))
        dev = hs.TopK(k); dev._load_device_state(m.sketch_views(out["sketches"])[top][r], n)
        assert list(dev._counters.items()) == list(mirror._counters.items()) and n > 300
        assert dev.top(3) == mirror.top(3) and dev.max_error() == mirror.max_error()


def test_host_side_add_equals_device_table_path():
    K = 60
    keys = np.random.RandomState(1).randint(0, K, size=500)
    h1, c1 = hs.HyperLogLog(precision=7, seed=3), hs.CountMinSketch(width=11, depth=4, seed=3)
    for k in keys:
        h1.add(int(k)); c1.add(int(k))
    ht, ct = hs.hll_table(7, 3, K), hs.cms_table(11, 4, 3, K)
    regs = np.zeros(128, np.uint8)
    np.maximum.at(regs, ht[0, keys], ht[1, keys].astype(np.uint8))
    cnt = np.zeros((4, 11), np.uint64)
    for row in range(4):
        np.add.at(cnt[row], ct[row, keys], 1)
    assert np.array_equal(h1._registers, regs) and np.array_equal(c1._counters, cnt)
    assert c1.estimate(int(keys[0])) >= int((keys == keys[0]).sum())     # never underestimates


def test_merge_contracts_over_replicas():
    m, kw, z = farm_model()
    out = O.oracle_run(m, O.make_params(n_replicas=5, seed=kw["seed"], end_ns=kw["end_ns"], rid_base=0))
    merged = D.merge_sketch_states(m, out["sketches"])
    views = m.sketch_views(out["sketches"])
    for i, v in views.items():
        if int(m.entities["i0"][i]) == A.HS_SK_HLL:
            acc = hs.HyperLogLog(precision=int(m.entities["i2"][i]))
            for r in range(5):
                o = hs.HyperLogLog(precision=int(m.entities["i2"][i])); o._load_device_state(v[r], 0); acc.merge(o)
            assert np.array_equal(acc._registers, merged[i])
        else:
            d, w = int(m.entities["i2"][i]), int(m.entities["i3"][i])
            acc = hs.CountMinSketch(w, d)
            for r in range(5):
                o = hs.CountMinSketch(w, d); o._load_device_state(v[r], int(out["entity_stats"][r][i]["c1"])); acc.merge(o)
            assert np.array_equal(acc._counters, merged[i])
            assert acc.item_count == int(out["entity_stats"][:, i]["c1"].sum())
    # Bloom (OR) and TopK (sequential, order dependent) over the replicas of the membership fixture
    m2, kw2, _ = G.load("philox_sketch_bloom_topk")
    out2 = O.oracle_run(m2, O.make_params(n_replicas=4, seed=kw2["seed"], end_ns=kw2["end_ns"], rid_base=0))
    merged2 = D.merge_sketch_states(m2, out2["sketches"])
    for i, v in m2.sketch_views(out2["sketches"]).items():
        e = m2.entities[i]
        if int(e["i0"]) == A.HS_SK_BLOOM:
            acc = hs.BloomFilter(int(e["i3"]), int(e["i2"]))
            for r in range(4):
                o = hs.BloomFilter(int(e["i3"]), int(e["i2"])); o._load_device_state(v[r], 1); acc.merge(o)
            assert np.array_equal(acc._bits, merged2[i]) and acc.item_count == 4
        else:
            acc = hs.TopK(int(e["i2"]))
            for r in range(4):
                o = hs.TopK(int(e["i2"])); o._load_device_state(v[r], int(out2["entity_stats"][r][i]["c1"])); acc.merge(o)
            assert merged2[i].top() == acc.top() and merged2[i].item_count == acc.item_count
    with pytest.raises(ValueError):
        hs.HyperLogLog(8).merge(hs.HyperLogLog(9))
    with pytest.raises(ValueError):
        hs.CountMinSketch(8, 2, seed=1).merge(hs.CountMinSketch(8, 2, seed=2))


def test_lowering_of_a_sketch_collector_model():
    K = 30
    hll = hs.HyperLogLog(precision=6, seed=4)
    col = hs.SketchCollector("uniques", hll, hs.KeyExtractor())
    srv = hs.Server("S", concurrency=1, service_time=hs.ExponentialLatency(0.01), downstream=col)
    src = hs.Source.poisson(rate=50.0, event_provider=hs.SimpleEventProvider(srv, context_fn=hs.UniformKeyContext(K)))
    model, objs = lowering.lower([src], [srv, col])
    i = objs.index(col)
    e = model.entities[i]
    assert int(e["kind"]) == A.HS_ENT_SKETCH and int(e["i0"]) == A.HS_SK_HLL and int(e["i2"]) == 6 and int(e["l0"]) == K
    assert np.array_equal(model.sketch_tables.reshape(2, K), hs.hll_table(6, 4, K))
    engine.validate_model(model)
    bad = hs.SketchCollector("x", hs.HyperLogLog(6), value_extractor=lambda ev: 1)
    with pytest.raises(hs.UnsupportedModelError, match="value_extractor"):
        lowering.lower([hs.Source.poisson(rate=1.0, event_provider=hs.SimpleEventProvider(bad, context_fn=hs.UniformKeyContext(K)))], [bad])


def test_lowering_of_topk_and_bloom_collectors():
    K = 20
    top = hs.TopKCollector("heavy", k=4)
    seen = hs.SketchCollector("seen", hs.BloomFilter.from_expected_items(100, 0.05, seed=2))
    s1 = hs.Server("A", service_time=hs.ExponentialLatency(0.01), downstream=top)
    s2 = hs.Server("B", service_time=hs.ExponentialLatency(0.01), downstream=seen)
    lb = hs.LoadBalancer("lb", backends=[s1, s2], strategy=hs.RoundRobin())
    src = hs.Source.poisson(rate=50.0, event_provider=hs.SimpleEventProvider(lb, context_fn=hs.UniformKeyContext(K)))
    model, objs = lowering.lower([src], [lb, s1, s2, top, seen])
    et, es = model.entities[objs.index(top)], model.entities[objs.index(seen)]
    assert int(et["i0"]) == A.HS_SK_TOPK and int(et["i2"]) == 4 and int(et["l0"]) == K
    bf = seen.sketch
    assert int(es["i0"]) == A.HS_SK_BLOOM and int(es["i3"]) == bf.size_bits == 624 and int(es["i2"]) == bf.num_hashes == 4
    assert np.array_equal(model.sketch_tables.reshape(4, K), hs.bloom_table(624, 4, 2, K))
    engine.validate_model(model)
    per, mer, total, mtotal = model.sketch_layout()
    assert total == (16 + 4 * 12) + 80 and mtotal == 80            # TOPK has no merged image


def test_lowering_of_a_quantile_estimator():
    est = hs.QuantileEstimator("p99", hs.LatencyExtractor(), compression=50.0)
    srv = hs.Server("S", concurrency=2, service_time=hs.ExponentialLatency(0.02), downstream=est)
    src = hs.Source.poisson(rate=40.0, target=srv)
    model, objs = lowering.lower([src], [srv, est])
    e = model.entities[objs.index(est)]
    assert int(e["kind"]) == A.HS_ENT_SKETCH and int(e["i0"]) == A.HS_SK_TDIGEST
    assert float(e["d0"]) == 50.0 and int(e["i2"]) == 100 and int(e["i3"]) == 200
    engine.validate_model(model)
    assert model.sketch_layout()[2:] == (32 + 200 * 16 + 800, 0)
    bad = hs.QuantileEstimator("x", value_extractor=lambda ev: 1.0)
    with pytest.raises(hs.UnsupportedModelError, match="LatencyExtractor"):
        lowering.lower([hs.Source.poisson(rate=1.0, target=bad)], [bad])
    model.entities[objs.index(est)]["i2"] = 99
    with pytest.raises(EngineError, match="buffer size"):
        engine.validate_model(model)
    assert est.summary()["count"] == 0 and est.summary()["p99"] == 0.0


def test_validation_rejects_bad_sketch_rows():
    def model(**over):
        b = hs.ModelBuilder()
        s = b.source(rate=1.0, key_population=8)
        h = b.sketch_hll(precision=5, table=hs.hll_table(5, 0, 8))
        b.set_target(s, h)
        m = b.build()
        for k, v in over.items():
            m.entities[k][1] = v
        return m
    engine.validate_model(model())
    for over, msg in ((dict(i2=3), "precision"), (dict(i0=9), "algorithm"), (dict(l0=-1), "population"), (dict(i1=5), "table")):
        with pytest.raises(EngineError, match=msg):
            engine.validate_model(model(**over))
    b = hs.ModelBuilder()
    s_ = b.source(rate=1.0, key_population=8)
    bl = b.sketch_bloom(size_bits=50, num_hashes=2, table=hs.bloom_table(50, 2, 0, 8))
    tk = b.sketch_topk(k=3, key_population=8)
    b.set_target(s_, bl)
    mb = b.build(); engine.validate_model(mb)
    mb.sketch_tables = mb.sketch_tables.copy(); mb.sketch_tables[9] = 50      # bit index == size_bits
    with pytest.raises(EngineError, match="Bloom bit"):
        engine.validate_model(mb)
    mb.sketch_tables[9] = 0; mb.entities[tk]["i2"] = 0
    with pytest.raises(EngineError, match="k must be positive"):
        engine.validate_model(mb)
    m = model()
    m.sketch_tables = m.sketch_tables.copy(); m.sketch_tables[3] = 32        # register index out of range for p = 5
    with pytest.raises(EngineError, match="HLL table"):
        engine.validate_model(m)


def test_device_hash_functions_equal_hashlib():
    """csrc/hs_sketch.h's SHA-256 based hashes (what a SKETCH row with K = 0 evaluates per event) against the
    host tables, which are hashlib evaluations of the reference's formulas -- small, large and edge keys."""
    L = O.lib()
    keys = list(range(0, 300)) + [999, 1000, 65535, 10**6, 123456789, 2**31 - 1]
    K = max(keys) + 1
    for p, seed in ((4, 0), (11, 7), (16, 2**40 + 5)):
        for k in keys:
            h = int.from_bytes(__import__("hashlib").sha256(__import__("struct").pack(">Q", seed) + repr(k).encode()).digest()[:8], "big")
            rest = h & ((1 << (64 - p)) - 1)
            i, r = C.c_int32(), C.c_int32()
            L.hs_cpu_hll_hash(seed, p, k, C.byref(i), C.byref(r))
            assert (i.value, r.value) == (h >> (64 - p), (64 - p) - rest.bit_length() + 1), (p, seed, k)
    small = [k for k in keys if k < 300]
    t = hs.hll_table(9, 3, 300)
    for k in small:
        i, r = C.c_int32(), C.c_int32(); L.hs_cpu_hll_hash(3, 9, k, C.byref(i), C.byref(r))
        assert (i.value, r.value) == (int(t[0, k]), int(t[1, k]))
    ct = hs.cms_table(272, 5, 11, 300)
    for row in range(5):
        rs = L.hs_cpu_cms_row_seed(11, row)
        assert [L.hs_cpu_cms_col(rs, 272, k) for k in small] == ct[row].tolist()
    bt = hs.bloom_table(9585, 7, 4, 300)
    for i in range(7):
        assert [L.hs_cpu_bloom_bit(4, i, 9585, k) for k in small] == bt[i].tolist()
    import hashlib, struct
    for k in (10**6, 2**31 - 1):       # large keys, large filter: the 128-bit (h1 + i h2) mod m of Python's ints
        for i in (0, 3, 6):
            dg = hashlib.sha256(struct.pack(">QQ", 9, i) + repr(k).encode()).digest()
            want = (int.from_bytes(dg[:8], "big") + i * int.from_bytes(dg[8:16], "big")) % (2**31 - 1)
            assert L.hs_cpu_bloom_bit(9, i, 2**31 - 1, k) == want


@pytest.mark.parametrize("name", ["philox_sketch_hll_direct", "philox_sketch_cms_farm", "philox_sketch_bloom_topk"])
def test_hashed_on_the_device_rows_give_the_reference_states(name):
    """The same fixtures with the per-key tables dropped (K = 0: SHA-256 per event): identical sketch states."""
    m, kw, z = G.load(name)
    b = hs.ModelBuilder()
    b._rows = [tuple(r) for r in m.entities.tolist()]; b._names = list(m.names)
    b._backends = [int(x) for x in m.backends]; b._key_table = m.key_table
    for i in m.ids_of(A.HS_ENT_SKETCH):
        e = m.entities[i]
        algo = int(e["i0"])
        if algo == A.HS_SK_TOPK:
            continue
        seed = int(z[f"sketch_seed_{i}"]); seed = 0 if seed < 0 else seed
        tmp = hs.ModelBuilder()
        if algo == A.HS_SK_HLL:
            tmp.sketch_hll(precision=int(e["i2"]), seed=seed)
        elif algo == A.HS_SK_CMS:
            tmp.sketch_cms(width=int(e["i3"]), depth=int(e["i2"]), seed=seed)
        else:
            tmp.sketch_bloom(size_bits=int(e["i3"]), num_hashes=int(e["i2"]), seed=seed)
        row = list(tmp._rows[0]); row[3] = sum(t.size for t in b._sketch_tables)     # i1: offset of the seed words
        b._sketch_tables.append(tmp._sketch_tables[0])
        b._rows[i] = tuple(row)
    hashed = b.build()
    assert all(int(hashed.entities["l0"][i]) == 0 for i in hashed.ids_of(A.HS_ENT_SKETCH) if int(hashed.entities["i0"][i]) != A.HS_SK_TOPK)
    engine.validate_model(hashed)
    out = O.oracle_run(hashed, O.make_params(n_replicas=1, **G.caps(z), **kw))
    assert hashed.sketch_tables.size < 40 and m.sketch_tables.size > 100
    assert out["sketches"][0].tobytes() == z["sketch_state"].tobytes()
    assert out["summaries"]["order_hash"][0] == z["summaries"]["order_hash"][0]


def test_write_back_of_sketch_states_onto_the_mirror_objects():
    """results.write_back with oracle outputs standing in for the device's (same layout): the INTEGRATION.md
    example -- TopKCollector, QuantileEstimator, HyperLogLog collector behind a consistent-hash ring, Zipf ids."""
    top = hs.TopKCollector("heavy", k=10)
    p99 = hs.QuantileEstimator("lat", hs.LatencyExtractor(), compression=100)
    seen = hs.SketchCollector("uniques", hs.HyperLogLog(precision=12, seed=1))
    servers = [hs.Server(f"S{i}", concurrency=2, service_time=hs.ExponentialLatency(0.02), downstream=d)
               for i, d in enumerate((top, p99, seen))]
    lb = hs.LoadBalancer("lb", backends=servers, strategy=hs.ConsistentHash(virtual_nodes=100))
    src = hs.Source.poisson(rate=120, event_provider=hs.SimpleEventProvider(lb, context_fn=hs.ZipfKeyContext(10_000, s=1.1)))
    sim = hs.Simulation(end_time=hs.Instant.from_seconds(30), sources=[src], entities=[lb, *servers, top, p99, seen])
    engine.validate_model(sim.model)
    out = O.oracle_run(sim.model, O.make_params(seed=1, end_ns=30 * 10**9, n_replicas=2))
    results.write_back(sim.model, sim.objects, out, 1, hs.Instant)
    i_top, i_p99, i_seen = (sim.objects.index(o) for o in (top, p99, seen))
    st = out["entity_stats"][1]
    assert top.events_processed == int(st[i_top]["c0"]) == top.total_count > 500
    assert top.top(1)[0].item == 0 and top.top(1)[0].count > 100          # rank 0 is the hottest id
    assert p99.sample_count == int(st[i_p99]["c1"]) and p99.summary()["count"] == p99.sample_count
    s = p99.summary()
    assert s["min"] <= s["p50"] <= s["p90"] <= s["p99"] <= s["p999"] <= s["max"]
    assert seen.events_processed == int(st[i_seen]["c0"]) and 100 < seen.sketch.cardinality() <= seen.sketch.item_count
    # the lowering hashes on the device above HASH_ON_DEVICE_ABOVE keys
    big = hs.SketchCollector("big", hs.HyperLogLog(precision=8, seed=3))
    src2 = hs.Source.poisson(rate=5, event_provider=hs.SimpleEventProvider(big, context_fn=hs.UniformKeyContext(lowering.HASH_ON_DEVICE_ABOVE + 1)))
    m2, objs2 = lowering.lower([src2], [big])
    e = m2.entities[objs2.index(big)]
    assert int(e["l0"]) == 0 and m2.sketch_tables.size == 2
    engine.validate_model(m2)
