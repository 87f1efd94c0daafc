"""Flat model table: the data format the engine (and the CPU oracle) consume.

A ``FlatModel`` is the lowered form of what ``Simulation.__init__`` receives as
``sources=`` / ``entities=`` (reference: happysimulator/core/simulation.py:66-102):
one ``hs_entity_desc`` row per Source / Server / Sink / Counter / LoadBalancer,
the LoadBalancer backend lists, an optional routing-key -> backend table (the
host-side evaluation of ConsistentHash.select, strategies.py:411-433) and an
optional per-cell parameter override for sweeps.  See include/hs_b200.h.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _abi as A


@dataclass
class FlatModel:
    entities: np.ndarray                      # ENTITY_DTYPE[n]
    names: list[str] = field(default_factory=list)
    backends: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    key_table: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    cell_d0: np.ndarray | None = None         # float64[n_cells, n]
    cell_i0: np.ndarray | None = None         # int32[n_cells, n]
    profiles: np.ndarray = field(default_factory=lambda: np.zeros(0, A.PROFILE_DTYPE))
    profile_table: np.ndarray = field(default_factory=lambda: np.zeros(0, np.float64))   # STEP profiles: breakpoints + rates
    sketch_tables: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    key_cdf: np.ndarray = field(default_factory=lambda: np.zeros(0, np.float64))
    outbox_cap: int = 0                       # linked partitions: cross-partition events a replica can emit per window
    inbox_cap: int = 0                        # ... and receive per barrier
    fault_events: list | None = None          # FAULT rows: the fault events whose `_cancelled` flags are re-read at run time

    @property
    def n_entities(self) -> int:
        return int(self.entities.shape[0])

    @property
    def n_cells(self) -> int:
        return 0 if self.cell_d0 is None else int(self.cell_d0.shape[0])

    # ---- SKETCH rows: state layout (the rule of csrc/hs_sketch.h, hs_sketch_layout) -------------
    def sketch_layout(self):
        """(per-replica offsets, merged offsets, bytes per replica, bytes of the merged image)."""
        per, mer, a, b = [0] * self.n_entities, [0] * self.n_entities, 0, 0
        for i in range(self.n_entities):
            e = self.entities[i]
            if int(e["kind"]) == A.HS_ENT_CACHE_SERVER:       # double insert_s[K + 1]; not merged
                per[i], mer[i] = a, b
                a += ((int(e["i0"]) + 1) * 8 + 15) // 16 * 16
                continue
            if int(e["kind"]) != A.HS_ENT_SKETCH:
                continue
            per[i], mer[i] = a, b
            if int(e["i0"]) == A.HS_SK_HLL:
                a += 1 << int(e["i2"]); b += 1 << int(e["i2"])
            elif int(e["i0"]) == A.HS_SK_BLOOM:
                nb = ((int(e["i3"]) + 63) // 64 * 8 + 15) // 16 * 16
                a += nb; b += nb
            elif int(e["i0"]) == A.HS_SK_TOPK:
                a += (16 + int(e["i2"]) * 12 + 15) // 16 * 16          # merged on the host: no merged image
            elif int(e["i0"]) == A.HS_SK_TDIGEST:
                a += 32 + int(e["i3"]) * 16 + (int(e["i2"]) * 8 + 15) // 16 * 16
            elif int(e["i0"]) == A.HS_SK_RESERVOIR:                      # hdr, mt[624], items[size]; host-merged
                a += 16 + 624 * 4 + (int(e["i2"]) * 4 + 15) // 16 * 16
            else:
                cells = int(e["i2"]) * int(e["i3"])
                a += (cells * 4 + 15) // 16 * 16; b += (cells * 8 + 15) // 16 * 16
        return per, mer, a, b

    def sketch_views(self, raw: np.ndarray) -> dict:
        """Per-replica states out of hs_outputs.sketches: {entity id: HLL uint8[n, 2^p] | CMS uint32[n, depth,
        width] | BLOOM uint64[n, words] | TOPK int64[n, 1 + 3 k] = (tracked, then item, count, error per slot) |
        RESERVOIR int64[n, 3 + 624 + size] = (items held, generator index, items seen, mt[624], the sample slots)}."""
        per = self.sketch_layout()[0]
        out = {}
        for i in self.ids_of(A.HS_ENT_SKETCH):
            e = self.entities[i]
            if int(e["i0"]) == A.HS_SK_HLL:
                out[i] = raw[:, per[i]: per[i] + (1 << int(e["i2"]))]
            elif int(e["i0"]) == A.HS_SK_BLOOM:
                nw = (int(e["i3"]) + 63) // 64
                out[i] = np.ascontiguousarray(raw[:, per[i]: per[i] + nw * 8]).view(np.uint64)
            elif int(e["i0"]) == A.HS_SK_TDIGEST:       # the raw bytes; see sketching.TDigest._load_device_state
                nb = 32 + int(e["i3"]) * 16 + (int(e["i2"]) * 8 + 15) // 16 * 16
                out[i] = np.ascontiguousarray(raw[:, per[i]: per[i] + nb])
            elif int(e["i0"]) == A.HS_SK_TOPK:
                k = int(e["i2"])
                hdr = np.ascontiguousarray(raw[:, per[i]: per[i] + 4]).view(np.uint32).astype(np.int64)
                sl = np.ascontiguousarray(raw[:, per[i] + 16: per[i] + 16 + 12 * k]).view(np.int32).astype(np.int64)
                out[i] = np.concatenate([hdr, sl], axis=1)
            elif int(e["i0"]) == A.HS_SK_RESERVOIR:
                size = int(e["i2"])
                hdr = np.ascontiguousarray(raw[:, per[i]: per[i] + 8]).view(np.uint32).astype(np.int64)
                tot = np.ascontiguousarray(raw[:, per[i] + 8: per[i] + 16]).view(np.int64)
                mt = np.ascontiguousarray(raw[:, per[i] + 16: per[i] + 16 + 2496]).view(np.uint32).astype(np.int64)
                it = np.ascontiguousarray(raw[:, per[i] + 2512: per[i] + 2512 + 4 * size]).view(np.int32).astype(np.int64)
                out[i] = np.concatenate([hdr, tot, mt, it], axis=1)
            else:
                d, w = int(e["i2"]), int(e["i3"])
                out[i] = np.ascontiguousarray(raw[:, per[i]: per[i] + d * w * 4]).view(np.uint32).reshape(-1, d, w)
        return out

    def cache_views(self, raw: np.ndarray) -> dict:
        """Per-replica TTL-cache states out of hs_outputs.sketches: {entity id: float64[n, K + 1] insertion times in
        seconds (0 = not cached; the last slot is the key-less "unknown" customer)}."""
        per = self.sketch_layout()[0]
        return {i: np.ascontiguousarray(raw[:, per[i]: per[i] + 8 * (int(self.entities[i]["i0"]) + 1)]).view(np.float64)
                for i in self.ids_of(A.HS_ENT_CACHE_SERVER)}

    def canonical_sketches(self, raw: np.ndarray) -> np.ndarray:
        """Copy of hs_outputs.sketches with the dead parts of TDIGEST rows zeroed (centroid slots past
        n_centroids and buffer slots past n_buffer keep leftovers of earlier merges; they are not state)."""
        raw = np.array(raw, dtype=np.uint8, copy=True).reshape(-1, self.sketch_layout()[2])
        per = self.sketch_layout()[0]
        for i in self.ids_of(A.HS_ENT_SKETCH):
            e = self.entities[i]
            if int(e["i0"]) != A.HS_SK_TDIGEST:
                continue
            cap, bsz = int(e["i3"]), int(e["i2"])
            for r in range(raw.shape[0]):
                n_c, n_b = (int(x) for x in raw[r, per[i]: per[i] + 8].view(np.uint32))
                raw[r, per[i] + 32 + n_c * 16: per[i] + 32 + cap * 16] = 0
                b0 = per[i] + 32 + cap * 16
                raw[r, b0 + n_b * 8: b0 + (bsz * 8 + 15) // 16 * 16] = 0
        return raw

    def merged_sketch_views(self, img: np.ndarray) -> dict:
        mer = self.sketch_layout()[1]
        out = {}
        for i in self.ids_of(A.HS_ENT_SKETCH):
            e = self.entities[i]
            if int(e["i0"]) == A.HS_SK_HLL:
                out[i] = img[mer[i]: mer[i] + (1 << int(e["i2"]))].copy()
            elif int(e["i0"]) == A.HS_SK_BLOOM:
                nw = (int(e["i3"]) + 63) // 64
                out[i] = img[mer[i]: mer[i] + nw * 8].copy().view(np.uint64)
            elif int(e["i0"]) in (A.HS_SK_TOPK, A.HS_SK_TDIGEST, A.HS_SK_RESERVOIR):
                continue
            else:
                d, w = int(e["i2"]), int(e["i3"])
                out[i] = img[mer[i]: mer[i] + d * w * 8].copy().view(np.uint64).reshape(d, w)
        return out

    def ids_of(self, kind: int) -> list[int]:
        return [i for i in range(self.n_entities) if int(self.entities["kind"][i]) == kind]

    def desc(self) -> A.ModelDesc:
        """ctypes view; keeps references to the numpy buffers on the returned struct."""
        ents = np.ascontiguousarray(self.entities)
        be = np.ascontiguousarray(self.backends, dtype=np.int32)
        kt = np.ascontiguousarray(self.key_table, dtype=np.int32)
        d = A.ModelDesc()
        d.abi_version = A.HS_ABI_VERSION
        d.n_entities = self.n_entities
        d.outbox_cap, d.inbox_cap = int(self.outbox_cap), int(self.inbox_cap)
        d.entities = ents.ctypes.data_as(C.POINTER(A.EntityDesc))
        d.n_backends = be.shape[0]
        d.key_population = kt.shape[0]
        d.backends = be.ctypes.data_as(C.POINTER(C.c_int32)) if be.size else None
        d.key_table = kt.ctypes.data_as(C.POINTER(C.c_int32)) if kt.size else None
        keep = [ents, be, kt]
        if self.cell_d0 is not None:
            cd = np.ascontiguousarray(self.cell_d0, dtype=np.float64)
            ci = np.ascontiguousarray(self.cell_i0, dtype=np.int32)
            assert cd.shape == ci.shape == (cd.shape[0], self.n_entities)
            d.n_cells = cd.shape[0]
            d.cell_d0 = cd.ctypes.data_as(C.POINTER(C.c_double))
            d.cell_i0 = ci.ctypes.data_as(C.POINTER(C.c_int32))
            keep += [cd, ci]
        if len(self.profile_table):                                  # STEP profile tables, PriorityQueue tables
            pt = np.ascontiguousarray(self.profile_table, dtype=np.float64)
            d.profile_table = pt.ctypes.data_as(C.POINTER(C.c_double))
            d.n_profile_table = pt.shape[0]
            keep.append(pt)
        if len(self.profiles):
            pr = np.array(self.profiles, dtype=A.PROFILE_DTYPE)          # a copy: p[2] of STEP rows is filled in below
            if len(self.profile_table):
                for row in pr:                                       # host address of the row's table, for the CPU oracle
                    if int(row["kind"]) == A.HS_PROF_STEP:
                        row["p"][2] = np.array([pt.ctypes.data + 8 * int(row["p"][0])], np.uint64).view(np.float64)[0]
            d.n_profiles = pr.shape[0]
            d.profiles = pr.ctypes.data
            keep.append(pr)
        if len(self.sketch_tables):
            st = np.ascontiguousarray(self.sketch_tables, dtype=np.int32)
            d.n_sketch_table = st.shape[0]
            d.sketch_tables = st.ctypes.data_as(C.POINTER(C.c_int32))
            keep.append(st)
        if len(self.key_cdf):
            kc = np.ascontiguousarray(self.key_cdf, dtype=np.float64)
            d.n_key_cdf = kc.shape[0]
            d.key_cdf = kc.ctypes.data_as(C.POINTER(C.c_double))
            keep.append(kc)
        d._keep = keep
        return d


class ModelBuilder:
    """Incremental construction of a FlatModel (entity ids are creation order)."""

    def __init__(self):
        self._rows: list[tuple] = []
        self._names: list[str] = []
        self._backends: list[int] = []
        self._key_table = np.zeros(0, np.int32)
        self._profiles: list[tuple] = []
        self._profile_tables: list[list[float]] = []
        self._sketch_tables: list[np.ndarray] = []
        self._key_cdf: list[np.ndarray] = []

    def _add(self, name, kind, target=-1, i0=0, i1=0, i2=0, l0=-1, d0=0.0, i3=0):
        self._rows.append((kind, target, i0, i1, i2, i3, l0, d0, 0.0))
        self._names.append(name)
        return len(self._rows) - 1

    def source(self, name="Source", *, rate=0.0, target=-1, poisson=True, stop_after_ns=-1, key_population=0,
               profile=None, key_cdf=None):
        """profile: None (ConstantRateProfile(rate)) or ("linear_ramp", duration_s, start_rate, end_rate)
        or ("spike", baseline_rate, spike_rate, warmup_s, spike_duration_s) or ("step", breakpoints, rates):
        n ascending breakpoints in seconds and n + 1 rates, rate(t) = rates[number of breakpoints <= t]."""
        i3 = 0
        if profile is not None and profile[0] == "step":
            breaks = [float(x) for x in profile[1]]
            rates = [float(x) for x in profile[2]]
            if len(rates) != len(breaks) + 1 or any(b <= a for a, b in zip(breaks, breaks[1:])):
                raise ValueError("step profile: n ascending breakpoints and n + 1 rates")
            off = sum(len(t) for t in self._profile_tables)
            self._profile_tables.append(breaks + rates)
            self._profiles.append((A.HS_PROF_STEP, 0, [float(off), float(len(breaks)), 0.0, 0.0]))
            i3 = len(self._profiles)
        elif profile is not None:
            kind = {"constant": A.HS_PROF_CONSTANT, "linear_ramp": A.HS_PROF_LINEAR_RAMP, "spike": A.HS_PROF_SPIKE}[profile[0]]
            ps = [float(x) for x in profile[1:]] + [0.0] * (5 - len(profile))
            self._profiles.append((kind, 0, ps))
            i3 = len(self._profiles)
        i2 = 0
        if key_cdf is not None:       # Zipf keys: the cumulative probabilities (lowering.zipf_cdf), zipf.py:96-123
            key_cdf = np.ascontiguousarray(key_cdf, dtype=np.float64)
            assert key_cdf.ndim == 1 and key_cdf.size == key_population
            i2 = 1 + sum(t.size for t in self._key_cdf)
            self._key_cdf.append(key_cdf)
        return self._add(name, A.HS_ENT_SOURCE, target, A.HS_ARR_POISSON if poisson else A.HS_ARR_CONSTANT,
                         key_population, i2, stop_after_ns, float(rate), i3=i3)

    def server(self, name="Server", *, concurrency=1, mean_service_s=0.01, exponential=True,
               downstream=-1, capacity=-1, lifo=False, priorities=None):
        """priorities: None (FIFOQueue, or LIFOQueue with lifo=True) or a PriorityQueue's table, one priority per
        routing key (floats; lower leaves first, ties in insertion order).  The table is appended to profile_table and
        the row's i3 is 1 + its offset there (include/hs_b200.h)."""
        pol, i3 = (A.HS_Q_LIFO if lifo else A.HS_Q_FIFO), 0
        if priorities is not None:
            if lifo:
                raise ValueError("a server has one queue policy: lifo or priorities")
            pol = A.HS_Q_PRIORITY
            i3 = 1 + sum(len(t) for t in self._profile_tables)
            self._profile_tables.append([float(x) for x in priorities])
        return self._add(name, A.HS_ENT_SERVER, downstream, int(concurrency), pol,
                         A.HS_SVC_EXPONENTIAL if exponential else A.HS_SVC_CONSTANT,
                         int(capacity), float(mean_service_s), i3=i3)

    def cache_server(self, name="CachingServer", *, key_slots, cache_ttl_s=30.0, cache_read_latency_s=0.0001,
                     datastore_read_latency_s=0.005, processing_latency_s=0.001, lifo=False):
        """examples/load-balancing/common.py:100-275 CachingServer: ``key_slots`` = K cache entries for keys 0..K-1
        (the cache must be larger than the key population, see include/hs_b200.h).  The delays are stored as the
        nanosecond counts the reference adds to `now`: int(delay_s * 1e9) (core/temporal.py:221-222)."""
        return self._add(name, A.HS_ENT_CACHE_SERVER, -1, int(key_slots), A.HS_Q_LIFO if lifo else A.HS_Q_FIFO,
                         int(cache_read_latency_s * 1e9), int(datastore_read_latency_s * 1e9), float(cache_ttl_s),
                         i3=int(processing_latency_s * 1e9))

    def sink(self, name="Sink"):
        return self._add(name, A.HS_ENT_SINK)

    def counter(self, name="Counter"):
        return self._add(name, A.HS_ENT_COUNTER)

    def probe(self, name="Probe", *, target, metric, interval_s):
        """instrumentation/probe.py:81-130: a Source ticking every `interval_s` through the GENERAL arrival
        path (its _ProbeProfile is not a ConstantRateProfile) whose payload samples `metric` of `target`.
        Returns (source_id, probe_id)."""
        pid = self._add(name + ".measure", A.HS_ENT_PROBE, int(target), A.METRICS[metric])
        sid = self.source(name, poisson=False, target=pid, profile=("constant", 1.0 / interval_s))
        return sid, pid

    @staticmethod
    def _seed_words(values) -> np.ndarray:
        """uint64 seeds as (lo, hi) int32 words: the table of a SKETCH row that hashes on the device (K = 0)."""
        v = np.array([int(x) & 0xFFFFFFFFFFFFFFFF for x in values], dtype=np.uint64)
        return np.ascontiguousarray(np.stack([v & np.uint64(0xFFFFFFFF), v >> np.uint64(32)], axis=1).astype(np.uint32)).view(np.int32).ravel()

    def _hashed_sketch(self, name, algo, i2, i3, words):
        off = sum(t.size for t in self._sketch_tables)
        self._sketch_tables.append(words)
        return self._add(name, A.HS_ENT_SKETCH, -1, algo, off, int(i2), 0, i3=int(i3))

    def sketch_hll(self, name="HLL", *, precision, table=None, seed=None):
        """SketchCollector(HyperLogLog(precision, seed)) on the routing key; table = hll_table(precision,
        seed, K): int32[2, K] (register index, run length) per key -- or table=None, seed=...: the device
        evaluates the SHA-256 hashes itself (any key population, no table)."""
        if table is None:
            return self._hashed_sketch(name, A.HS_SK_HLL, precision, 0, self._seed_words([seed or 0]))
        table = np.ascontiguousarray(table, dtype=np.int32)
        assert table.ndim == 2 and table.shape[0] == 2
        off = sum(t.size for t in self._sketch_tables)
        self._sketch_tables.append(table)
        return self._add(name, A.HS_ENT_SKETCH, -1, A.HS_SK_HLL, off, int(precision), table.shape[1])

    def sketch_cms(self, name="CMS", *, width, depth, table=None, seed=None):
        """SketchCollector(CountMinSketch(width, depth, seed)) on the routing key; table = cms_table(width,
        depth, seed, K): int32[depth, K], the column of key k in each row -- or table=None, seed=...: hashed on the
        device; the row seeds sha256(pack(">QQ", seed, row))[:8] (count_min_sketch.py:136-143) travel instead."""
        if table is None:
            import hashlib, struct
            rs = [int.from_bytes(hashlib.sha256(struct.pack(">QQ", seed or 0, row)).digest()[:8], "big") for row in range(depth)]
            return self._hashed_sketch(name, A.HS_SK_CMS, depth, width, self._seed_words(rs))
        table = np.ascontiguousarray(table, dtype=np.int32)
        assert table.ndim == 2 and table.shape[0] == depth
        off = sum(t.size for t in self._sketch_tables)
        self._sketch_tables.append(table)
        return self._add(name, A.HS_ENT_SKETCH, -1, A.HS_SK_CMS, off, int(depth), table.shape[1], i3=int(width))

    def sketch_bloom(self, name="Bloom", *, size_bits, num_hashes, table=None, seed=None):
        """SketchCollector(BloomFilter(size_bits, num_hashes, seed)) on the routing key; table =
        bloom_table(size_bits, num_hashes, seed, K): int32[num_hashes, K], the bit each hash sets for key k -- or
        table=None, seed=...: hashed on the device."""
        if table is None:
            return self._hashed_sketch(name, A.HS_SK_BLOOM, num_hashes, size_bits, self._seed_words([seed or 0]))
        table = np.ascontiguousarray(table, dtype=np.int32)
        assert table.ndim == 2 and table.shape[0] == num_hashes
        off = sum(t.size for t in self._sketch_tables)
        self._sketch_tables.append(table)
        return self._add(name, A.HS_ENT_SKETCH, -1, A.HS_SK_BLOOM, off, int(num_hashes), table.shape[1], i3=int(size_bits))

    def sketch_tdigest(self, name="TDigest", *, compression=100.0, capacity=None):
        """QuantileEstimator(compression) on the request's latency in seconds (tdigest.py:47; buffer of
        int(compression * 2) values, flushed into at most `capacity` centroids, default 4 x compression)."""
        buf = int(float(compression) * 2)
        cap = int(capacity) if capacity is not None else 2 * buf
        return self._add(name, A.HS_ENT_SKETCH, -1, A.HS_SK_TDIGEST, 0, buf, 1, d0=float(compression), i3=cap)

    def sketch_topk(self, name="TopK", *, k, key_population):
        """TopKCollector(k) / SketchCollector(TopK(k)) on the routing key (Space-Saving; no table)."""
        return self._add(name, A.HS_ENT_SKETCH, -1, A.HS_SK_TOPK, 0, int(k), int(key_population))

    def sketch_reservoir(self, name="Reservoir", *, size, key_population, seed=None, state=None):
        """SketchCollector(ReservoirSampler(size, seed)) on the routing key (reservoir.py:30).  The row's table is
        the MT19937 state the sampler starts from: ``state`` = random.Random.getstate()[1] (625 words), or the
        state of random.Random(seed)."""
        if state is None:
            import random
            state = random.Random(seed).getstate()[1]
        words = np.array([int(x) for x in state], dtype=np.uint32).view(np.int32)
        assert words.size == 625
        off = sum(t.size for t in self._sketch_tables)
        self._sketch_tables.append(words)
        return self._add(name, A.HS_ENT_SKETCH, -1, A.HS_SK_RESERVOIR, off, int(size), int(key_population))

    def remote(self, name="Remote", *, link, dest_entity):
        """Stand-in for an entity of another partition (HS_ENT_REMOTE): events sent to it leave through the
        partition's outgoing link number ``link`` and arrive at entity ``dest_entity`` of the link's destination."""
        return self._add(name, A.HS_ENT_REMOTE, -1, int(link), int(dest_entity))

    def load_balancer(self, name="LB", *, backends, key_table=None):
        off = len(self._backends)
        self._backends += [int(b) for b in backends]
        strat = A.HS_LB_ROUND_ROBIN
        if key_table is not None:
            strat = A.HS_LB_KEY_TABLE
            self._key_table = np.asarray(key_table, dtype=np.int32)
        return self._add(name, A.HS_ENT_LB, -1, strat, off, len(backends))

    def fault(self, name="Fault", *, target, time_ns, crash, sort_index, cancelled=False):
        """One event of a node fault (HS_ENT_FAULT, faults/node_faults.py CrashNode / PauseNode): at ``time_ns`` it sets
        (``crash``) or clears the crashed flag of entity ``target``.  ``sort_index`` is the event's bootstrap sort index
        (sources, then probes, then the faults in schedule order); ``cancelled``: its FaultHandle was cancelled.  FAULT
        rows must come after every other row."""
        return self._add(name, A.HS_ENT_FAULT, int(target), 0, 1 if crash else 0, 1 if cancelled else 0, int(time_ns),
                         i3=int(sort_index))

    def set_target(self, ent, target):
        r = list(self._rows[ent]); r[1] = int(target); self._rows[ent] = tuple(r)

    def build(self) -> FlatModel:
        ents = np.array(self._rows, dtype=A.ENTITY_DTYPE)
        m = FlatModel(entities=ents, names=list(self._names),
                      backends=np.asarray(self._backends, dtype=np.int32),
                      key_table=self._key_table)
        if self._profiles:
            m.profiles = np.array(self._profiles, dtype=A.PROFILE_DTYPE)
        if self._profile_tables:
            m.profile_table = np.array([x for t in self._profile_tables for x in t], dtype=np.float64)
        if self._sketch_tables:
            m.sketch_tables = np.concatenate([t.ravel() for t in self._sketch_tables]).astype(np.int32)
        if self._key_cdf:
            m.key_cdf = np.concatenate(self._key_cdf).astype(np.float64)
        return m


# ---- the BASELINE.json configurations ------------------------------------

def mm1(rate=8.0, mean_service_s=0.1, *, poisson=True, exponential=True, capacity=-1,
        concurrency=1, lifo=False) -> FlatModel:
    """configs[0]/[1]: Source.poisson(rate) -> Server(Exponential(mean)) -> Sink."""
    b = ModelBuilder()
    src = b.source(rate=rate, poisson=poisson)
    srv = b.server(concurrency=concurrency, mean_service_s=mean_service_s, exponential=exponential,
                   capacity=capacity, lifo=lifo)
    snk = b.sink()
    b.set_target(src, srv)
    b.set_target(srv, snk)
    return b.build()


def lb_round_robin(n_servers=64, rate=512.0, mean_service_s=0.1) -> FlatModel:
    """configs[2]: Source.poisson(rate) -> LoadBalancer(RoundRobin) -> n x Server(1, Exp) -> Sink."""
    b = ModelBuilder()
    src = b.source(rate=rate)
    servers = [b.server(f"S{i}", mean_service_s=mean_service_s) for i in range(n_servers)]
    snk = b.sink()
    lb = b.load_balancer(backends=servers)
    b.set_target(src, lb)
    for s in servers:
        b.set_target(s, snk)
    return b.build()


def lb_key_table(key_table, n_servers, rate, mean_service_s=0.1) -> FlatModel:
    """configs[3]: Source.poisson(rate) with client_id ~ Uniform{0..K-1} ->
    LoadBalancer(ConsistentHash) -> n x Server -> Sink; key_table[k] = backend slot
    (use lowering.consistent_hash_table to evaluate the MD5 ring on the host)."""
    b = ModelBuilder()
    src = b.source(rate=rate, key_population=len(key_table))
    servers = [b.server(f"S{i}", mean_service_s=mean_service_s) for i in range(n_servers)]
    snk = b.sink()
    lb = b.load_balancer(backends=servers, key_table=key_table)
    b.set_target(src, lb)
    for s in servers:
        b.set_target(s, snk)
    return b.build()


def mmc_sweep(cs=range(1, 33), rhos=(0.5, 0.6, 0.7, 0.8, 0.85, 0.9, 0.95, 0.99), mu=10.0) -> FlatModel:
    """configs[4]: M/M/c cells, c x rho grid, lambda = rho * c * mu (SURVEY.md 8(d).5)."""
    m = mm1(rate=1.0, mean_service_s=1.0 / mu)
    cells = [(c, rho) for c in cs for rho in rhos]
    n = m.n_entities
    cd = np.tile(m.entities["d0"].astype(np.float64), (len(cells), 1))
    ci = np.tile(m.entities["i0"].astype(np.int32), (len(cells), 1))
    for k, (c, rho) in enumerate(cells):
        cd[k, 0] = rho * c * mu
        ci[k, 1] = c
    m.cell_d0, m.cell_i0 = cd, ci
    m.cells = cells
    return m
