"""The models and helpers the linked sweep tests share: linked runs whose replicas are sweep cells (their oracle is
tests/layered_oracle_lib.py).  Test infrastructure."""
from __future__ import annotations

import dataclasses

import numpy as np

from happysim_b200 import _abi as A
from happysim_b200.engine import make_params


def partition_params(lm, *, seed, end_ns, n, caps, seed_stride=0, rid_stride=None, replica_index_base=0, replicas_per_cell=1,
                     flags=A.HS_RUN_ORDER_HASH):
    """The hs_run_params of every partition of a linked run, as LinkedRun.run makes them (partition q: word q + g * rid_stride)."""
    nP = lm.n_partitions
    rs = nP + 1 if rid_stride is None else rid_stride
    return [make_params(seed=seed, seed_stride=seed_stride, end_ns=end_ns, n_replicas=n, rid_base=q, rid_stride=rs,
                        replica_index_base=replica_index_base, replicas_per_cell=replicas_per_cell, flags=flags,
                        **(caps[q] if isinstance(caps, (list, tuple)) else caps)) for q in range(nP)]


def cell_of(n, replica_index_base=0, replicas_per_cell=1, n_cells=1):
    return ((replica_index_base + np.arange(n)) // replicas_per_cell) % n_cells


# ---- models ---------------------------------------------------------------------------------------------------------------

def with_link_cells(lm, rng, n_cells: int, zero_loss_cell: bool = True):
    """``lm`` (partitions possibly with model cells already) with a per-cell link table: cell 0 keeps the links'
    own values, every other cell scales each latency mean by 0.5 to 2 and draws a loss from {0, 0.05, 0.2}; with
    ``zero_loss_cell`` cell 1 loses nothing and cell 2 (if any) loses on every link, so lossless and lossy cells sit
    side by side."""
    tab = []
    for q, ls in enumerate(lm.links):
        t = np.zeros((n_cells, len(ls), 2), np.float64)
        for k, l in enumerate(ls):
            t[0, k] = (l.latency_mean_s, l.packet_loss)
            for c in range(1, n_cells):
                loss = float(rng.choice([0.0, 0.05, 0.2]))
                if zero_loss_cell and c == 1:
                    loss = 0.0
                elif zero_loss_cell and c == 2:
                    loss = 0.2
                t[c, k] = (l.latency_mean_s * float(rng.uniform(0.5, 2.0)), loss)
        tab.append(t)
    return dataclasses.replace(lm, models=list(lm.models), links=[list(ls) for ls in lm.links], cell_links=tab)


def with_model_cells(lm, rng, n_cells: int):
    """``lm`` whose every partition has ``n_cells`` model cells (tests/sweep_models.with_cells, REMOTE rows untouched)."""
    import sweep_models as SM
    return dataclasses.replace(lm, models=[SM.with_cells(m, rng, n_cells, "any") for m in lm.models])


def celled(lm, seed: int, n_cells: int):
    """A LinkedModel with ``n_cells`` cells in the partitions and on the links."""
    rng = np.random.RandomState(31_000 + seed)
    return with_link_cells(with_model_cells(lm, rng, n_cells), rng, n_cells)


KEYS = ("summaries", "entity_stats", "records", "sink_samples", "service_samples", "sketches")


def assert_replica_equal(got, want, r_got: int, r_want: int, what=""):
    """Replica r_got of one linked run's outputs against replica r_want of another's, partition by partition, byte
    for byte.  Recorder rings of different capacities (runs sized for different rates) are compared over the slots
    both have, which must hold everything the replica recorded."""
    rings = {"records": "events_processed", "sink_samples": "n_sink_samples", "service_samples": "n_service_samples"}
    for q, (g, w) in enumerate(zip(got, want)):
        for k in KEYS:
            a, b = g.get(k), w.get(k)
            if a is None and b is None:
                continue
            x, y = a[r_got], b[r_want]
            if k in rings and x.shape != y.shape:
                m = min(len(x), len(y))
                if k != "records":
                    assert int(g["summaries"][rings[k]][r_got]) <= m, f"{what}: partition {q}, {k} wrapped"
                x, y = x[:m], y[:m]
            assert x.tobytes() == y.tobytes(), f"{what}: partition {q}, {k} of replica {r_got} differs"
