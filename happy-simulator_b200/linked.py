"""Partitions joined by PartitionLinks (SURVEY.md 8(f) row 4, first half): the data model of a linked run.

Reference: parallel/simulation.py:31-284 (one Simulation per partition), parallel/routing.py:17-63 (the router that
moves events aimed at another partition into an outbox), parallel/coordinator.py:75-227 (windows of
min(link.min_latency), barrier, exchange with loss / latency override).

Here a partition is a FlatModel of its own in which every entity of ANOTHER partition that it sends to appears as an
HS_ENT_REMOTE row (link slot, entity id over there); the coordinator's window ends are computed on the host, in the
float arithmetic of coordinator.py:88-95, and every partition runs window after window with
``hs_run(end_ns=window end, resume=window > 0)``; ``hs_coordinator_exchange`` moves the outboxes at each barrier."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field

import numpy as np

from . import _abi as A
from .model import FlatModel


@dataclass(frozen=True)
class LinkSpec:
    """One outgoing link of a partition, as the engine sees it (hs_link_desc + the partition it ends in)."""
    dest: int                       # index of the destination partition
    latency_kind: int               # HS_SVC_CONSTANT | HS_SVC_EXPONENTIAL
    latency_mean_s: float
    packet_loss: float = 0.0
    stream: int = 0                 # id of the latency object (shared objects share their draw counter)


@dataclass
class LinkedModel:
    models: list[FlatModel]
    names: list[str]
    links: list[list[LinkSpec]]     # links[p][slot]
    window_s: float
    n_streams: int = 1
    objects: list[list] = field(default_factory=list)     # per partition: entity id -> user object (lowering)
    # sweep cells: per partition float64 [n_cells, slot, 2], every link's (latency_mean_s, packet_loss) in every cell;
    # the partitions' models carry the cells' rows (FlatModel.cell_d0 / cell_i0).  None: one configuration, ``links``.
    cell_links: list[np.ndarray] | None = None

    @property
    def n_partitions(self) -> int:
        return len(self.models)

    @property
    def n_cells(self) -> int:
        """Sweep cells of the run (0: none).  Replica g runs cell (g / replicas_per_cell) % n_cells everywhere."""
        return 0 if self.cell_links is None else int(self.cell_links[0].shape[0])

    @classmethod
    def from_cells(cls, cells: list["LinkedModel"]) -> "LinkedModel":
        """One LinkedModel whose cell c is ``cells[c]``: models, links and windows of one linked topology (the caller
        checks that), differing at most in the models' d0 / server i0 and the links' latency mean and loss."""
        lead = cells[0]
        models = []
        for q, m in enumerate(lead.models):
            mm = dataclasses.replace(m, cell_d0=np.stack([np.asarray(c.models[q].entities["d0"], np.float64) for c in cells]),
                                     cell_i0=np.stack([np.asarray(c.models[q].entities["i0"], np.int32) for c in cells]))
            mm.outbox_cap = max(int(c.models[q].outbox_cap) for c in cells)
            mm.inbox_cap = max(int(c.models[q].inbox_cap) for c in cells)
            models.append(mm)
        tab = [np.array([[(float(l.latency_mean_s), float(l.packet_loss)) for l in c.links[q]] for c in cells],
                        np.float64).reshape(len(cells), len(lead.links[q]), 2) for q in range(lead.n_partitions)]
        return cls(models, list(lead.names), [list(ls) for ls in lead.links], window_s=lead.window_s,
                   n_streams=lead.n_streams, objects=lead.objects, cell_links=tab)

    def cell(self, c: int) -> "LinkedModel":
        """The plain LinkedModel (no cells) of cell ``c``: its rows written into the models, its link parameters."""
        if not self.n_cells:
            return self
        models = []
        for m in self.models:
            E = m.entities.copy()
            E["d0"], E["i0"] = m.cell_d0[c], m.cell_i0[c]
            models.append(dataclasses.replace(m, entities=E, cell_d0=None, cell_i0=None))
        links = [[dataclasses.replace(l, latency_mean_s=float(t[c, k, 0]), packet_loss=float(t[c, k, 1]))
                  for k, l in enumerate(ls)] for ls, t in zip(self.links, self.cell_links)]
        return LinkedModel(models, list(self.names), links, window_s=self.window_s, n_streams=self.n_streams,
                           objects=self.objects)

    def window_ends(self, end_ns: int, start_ns: int = 0) -> list[int]:
        """WindowedCoordinator.run's window ends (coordinator.py:86-96): float seconds, clamped to the end time,
        converted back with Instant.from_seconds (truncation)."""
        ends, cur = [], int(start_ns)
        end_s = float(end_ns) / 1_000_000_000
        while cur < end_ns:
            w = float(cur) / 1_000_000_000 + self.window_s
            if w > end_s:
                w = end_s
            nxt = int(w * 1_000_000_000)
            if nxt <= cur:
                # e.g. an end time whose nanoseconds do not survive the trip through float seconds: the clamped window
                # ends 1 ns short of it, for ever -- the reference's coordinator never returns from such a run
                raise ValueError(f"window of {self.window_s} s does not advance the clock at {cur} ns (end {end_ns} ns): "
                                 "the reference's WindowedCoordinator would loop for ever")
            ends.append(nxt)
            cur = nxt
        return ends

    def link_descs(self, p: int):
        """(ctypes hs_link_desc array, destination partition indices) of partition p's outgoing links.  With cells the
        array is the per-cell table [n_cells][slot] of hs_coordinator_exchange_cells."""
        ls = self.links[p]
        nc = max(1, self.n_cells)
        arr = (A.LinkDesc * max(1, nc * len(ls)))()
        for c in range(nc):
            for k, l in enumerate(ls):
                d = arr[c * len(ls) + k]
                d.latency_kind, d.stream = int(l.latency_kind), int(l.stream)
                if self.n_cells:
                    d.latency_mean_s, d.packet_loss = (float(v) for v in self.cell_links[p][c, k])
                else:
                    d.latency_mean_s, d.packet_loss = float(l.latency_mean_s), float(l.packet_loss)
        return arr, [int(l.dest) for l in ls]

    def validate(self) -> None:
        for p, ls in enumerate(self.links):
            for l in ls:
                if not 0 <= l.dest < self.n_partitions or l.dest == p:
                    raise ValueError("link destination out of range")
                if self.models[l.dest].inbox_cap <= 0:
                    raise ValueError(f"partition {self.names[l.dest]!r} is a link destination but has no inbox")
                if not 0 <= l.stream < self.n_streams:
                    raise ValueError("latency stream id out of range")
        for p, m in enumerate(self.models):
            for i in m.ids_of(A.HS_ENT_REMOTE):
                slot, dst_ent = int(m.entities["i0"][i]), int(m.entities["i1"][i])
                if not 0 <= slot < len(self.links[p]):
                    raise ValueError(f"partition {self.names[p]!r}: REMOTE row {i} uses link slot {slot} of {len(self.links[p])}")
                dm = self.models[self.links[p][slot].dest]
                if not 0 <= dst_ent < dm.n_entities or int(dm.entities["kind"][dst_ent]) in (A.HS_ENT_SOURCE, A.HS_ENT_PROBE, A.HS_ENT_REMOTE):
                    raise ValueError(f"partition {self.names[p]!r}: REMOTE row {i} points at entity {dst_ent} of "
                                     f"{self.names[self.links[p][slot].dest]!r}, which cannot receive requests")
            if m.ids_of(A.HS_ENT_REMOTE) and m.outbox_cap <= 0:
                raise ValueError(f"partition {self.names[p]!r} has REMOTE rows but no outbox")
        if self.cell_links is not None:
            nc = self.n_cells
            for p, (m, t) in enumerate(zip(self.models, self.cell_links)):
                if t.shape != (nc, len(self.links[p]), 2) or m.n_cells != nc:
                    raise ValueError(f"partition {self.names[p]!r}: {m.n_cells} model cells and a link table of shape "
                                     f"{t.shape}, the run has {nc} cells of {len(self.links[p])} links")
                if not ((t[..., 0] >= 0).all() and (t[..., 1] >= 0).all() and (t[..., 1] < 1).all()):
                    raise ValueError(f"partition {self.names[p]!r}: a cell's link latency is < 0 or its loss outside [0, 1)")


class LinkedRun:
    """A LinkedModel on one GPU: one engine per partition (the same replicas in each), one coordinator.

    ``run()`` is WindowedCoordinator.run (coordinator.py:75-172): for every window, every partition runs
    ``hs_run(end_ns=window end, resume=window > 0, HS_RUN_LINKED)``, then ``hs_coordinator_exchange`` drains the
    partitions' outboxes in partition order.  Replica r of partition q draws from the Philox replica word
    ``q + g * (P + 1)`` (g = global replica index), the coordinator from ``P + g * (P + 1)``."""

    def __init__(self, lm: LinkedModel, *, device: int = 0):
        from . import engine as _engine
        import torch
        lm.validate()
        self.lm, self.device = lm, device
        # one CUDA stream for every partition and the coordinator: the window loop (partitions x windows launches plus the
        # barrier kernels) is queued without a host synchronisation in between
        self._stream = torch.cuda.Stream(device=device) if torch.cuda.is_available() else None
        sp = self._stream.cuda_stream if self._stream is not None else None
        self._stream_ptr = sp
        self.engines = [_engine.Engine(device, stream=sp) for _ in lm.models]
        for e, m in zip(self.engines, lm.models):
            e.upload(m, partition=True)
        self.coordinator = None
        self.windows = 0

    def close(self):
        for e in self.engines:
            e.close()
        if self.coordinator is not None:
            self.coordinator.close()

    def run(self, *, seed, end_ns, n_replicas=1, replica_index_base=0, caps=None, flags=A.HS_RUN_ORDER_HASH, queue_ring=0,
            buckets=None, bucket_sample_cap=0, replicas_per_cell=1, seed_stride=0, rid_stride=None):
        """caps: per-partition dicts of record_cap / sample_cap / service_cap (or one dict for all).  Returns the
        per-partition outputs (Engine.read_outputs) and (delivered, lost, overflowed) per replica.

        Replica g draws with Philox key ``seed + g * seed_stride``; partition q with replica word ``q + g * rid_stride``,
        the coordinator with ``P + g * rid_stride`` (rid_stride defaults to P + 1).  With cells (``LinkedModel.n_cells``)
        replica g runs cell (g / replicas_per_cell) % n_cells in every partition and at every barrier, and every
        partition's outputs get ``cell_totals`` (Engine.read_cell_totals).

        ``buckets=(width_s, n)`` (checked by the caller, with no recorder rings in ``caps``) buckets the samples of
        every partition that has a Sink, tracker or Probe row; ``bucket_sample_cap`` > 0 adds their p50 / p99.  Those
        partitions' outputs get the keys of ``buckets.read_outputs``; the other partitions run as without buckets."""
        from . import buckets as _buckets
        from . import engine as _engine
        lm, nP = self.lm, self.lm.n_partitions
        nc = lm.n_cells
        rs = nP + 1 if rid_stride is None else int(rid_stride)
        if self.coordinator is not None:
            self.coordinator.close()
        self.coordinator = _engine.Coordinator(self.device, n_replicas, lm.n_streams, seed=seed, seed_stride=seed_stride,
                                               rid_base=nP, rid_stride=rs, replica_index_base=replica_index_base,
                                               stream=self._stream_ptr)
        caps = caps or {}
        link_args = [lm.link_descs(q) for q in range(nP)]
        ends = lm.window_ends(end_ns)
        bucketed = [q for q, m in enumerate(lm.models) if buckets is not None and _buckets.rows(m)]
        try:
            for q in bucketed:
                self.engines[q].set_buckets(*buckets)
                self.engines[q].set_bucket_percentiles(bucket_sample_cap)
            for w, wend in enumerate(ends):
                for q, e in enumerate(self.engines):
                    c = caps[q] if isinstance(caps, (list, tuple)) else caps
                    e.run(_engine.make_params(seed=seed, seed_stride=seed_stride, end_ns=wend, n_replicas=n_replicas,
                                              rid_base=q, rid_stride=rs, replica_index_base=replica_index_base,
                                              replicas_per_cell=replicas_per_cell, engine=3, resume=1 if w else 0,
                                              flags=flags | A.HS_RUN_LINKED, queue_ring=queue_ring, **c))
                for q, e in enumerate(self.engines):
                    arr, dst = link_args[q]
                    if dst:
                        self.coordinator.exchange(e, arr, [self.engines[d] for d in dst], nc, replicas_per_cell)
            self.windows = len(ends)
            outs = [e.read_outputs() for e in self.engines]
            if nc:
                for o, e in zip(outs, self.engines):
                    o["cell_totals"] = e.read_cell_totals(nc)
            for q in bucketed:
                objs = lm.objects[q] if lm.objects else [None] * lm.models[q].n_entities
                outs[q].update(_buckets.read_outputs(self.engines[q], buckets, bucket_sample_cap, lm.models[q], objs,
                                                     max(1, nc)))
        finally:
            for e in self.engines:          # the engines may run again without buckets
                e.set_bucket_percentiles(0)
                e.set_buckets(0.0, 0)
        return outs, self.coordinator.read()
