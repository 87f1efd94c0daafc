"""Linked ParallelSimulations whose partitions carry node-fault schedules (CrashNode, PauseNode): the FAULT rows a
partition's schedule lowers to, and the random models of tests/golden/random_linked_faults.npz.  Test infrastructure.

A fault is given as (class, entity name, t0_s, t1_s, cancelled): ("crash", name, at, restart_at or None) or
("pause", name, start, end).  Every partition's Simulation bootstraps its own schedule after its sources and probes
with its own event counter (core/simulation.py:77,162-169), so a partition's fault events take the sort indices
n_sources + 0, 1, 2, ... whatever the other partitions hold."""
from __future__ import annotations

import dataclasses

import numpy as np

from happysim_b200 import _abi as A


def from_seconds(t_s) -> int:
    """Instant.from_seconds, as lowering.fault_events applies it"""
    return t_s * 1_000_000_000 if isinstance(t_s, int) else int(t_s * 1_000_000_000)


def fault_rows(model, faults):
    """The FAULT rows (ENTITY_DTYPE tuples) and names of a partition's schedule ``faults``."""
    names = list(model.names)
    k = int((model.entities["kind"] == A.HS_ENT_SOURCE).sum())      # the sources' (and probes' ticks') first events
    rows, rnames = [], []
    for cls, name, t0, t1, cancelled in faults:
        tgt = names.index(name)
        for t_s, crash in ([(t0, True)] + ([] if t1 is None else [(t1, False)])) if cls == "crash" else [(t0, True), (t1, False)]:
            rows.append((A.HS_ENT_FAULT, tgt, 0, int(crash), int(bool(cancelled)), k, from_seconds(t_s), 0.0, 0.0))
            rnames.append(f"fault:{name}")
            k += 1
    return rows, rnames


def with_faults(model, faults):
    """``model`` with the FAULT rows of ``faults`` appended (a copy; outbox / inbox capacities kept)."""
    rows, rnames = fault_rows(model, faults)
    if not rows:
        return model
    m = dataclasses.replace(model, entities=np.concatenate([model.entities, np.array(rows, dtype=A.ENTITY_DTYPE)]),
                            names=list(model.names) + rnames)
    m.outbox_cap, m.inbox_cap = model.outbox_cap, model.inbox_cap
    return m


def linked_with_faults(lm, schedules):
    """A LinkedModel whose partition q holds the FAULT rows of ``schedules[q]``."""
    from happysim_b200.linked import LinkedModel
    return LinkedModel([with_faults(m, s) for m, s in zip(lm.models, schedules)], list(lm.names), lm.links,
                       window_s=lm.window_s, n_streams=lm.n_streams)


RANDOM_SEEDS = 48


def random_schedules(lm, end_s, seed: int):
    """0-3 node faults per partition on its own entities (never a REMOTE row): crashes with and without a restart,
    pauses, some overlapping, some beyond end_time, about one in six cancelled.  Times on a 1 ms grid."""
    rng = np.random.RandomState(90_000 + seed)
    out = []
    for m in lm.models:
        cand = [m.names[i] for i in range(m.n_entities) if int(m.entities["kind"][i]) != A.HS_ENT_REMOTE]
        faults = []
        for _ in range(int(rng.choice([0, 1, 2, 2, 3]))):
            name = str(rng.choice(cand))
            t0 = round(float(rng.uniform(0.0, end_s * 0.9)), 3)
            t1 = round(t0 + float(rng.uniform(0.05, end_s * 0.6)), 3)
            cls = "pause" if rng.rand() < 0.35 else "crash"
            if cls == "crash" and rng.rand() < 0.3:
                t1 = None
            faults.append((cls, name, t0, t1, bool(rng.rand() < 0.17)))
        out.append(faults)
    return out


def random_linked_fault_model(seed: int):
    """tests/random_models.random_linked_model(seed) with random_schedules -> (LinkedModel with FAULT rows, end_s,
    description, schedules)"""
    import random_models as RM
    lm, end_s, what = RM.random_linked_model(seed)
    sch = random_schedules(lm, end_s, seed)
    return linked_with_faults(lm, sch), end_s, what + f", {sum(len(s) for s in sch)} faults", sch


ROW = np.dtype([("seed", "<i4"), ("part", "<i4"), ("events_processed", "<i8"), ("final_time_ns", "<i8"), ("order_hash", "<u8"),
                ("heap_left", "<i4"), ("n_sink_samples", "<i8"), ("n_service_samples", "<i8"), ("stats_digest", "<u8"),
                ("events_cancelled", "<i8"), ("tie", "<i4")])
TOP = np.dtype([("seed", "<i4"), ("windows", "<i4"), ("delivered", "<i8"), ("total_events", "<i8")])


def digest(a) -> int:
    import hashlib
    return int.from_bytes(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()[:8], "little")
