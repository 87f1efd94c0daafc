"""Time buckets of an ensemble's Sink / LatencyTracker / ThroughputTracker / Probe samples.

``Simulation.run_ensemble(..., buckets=(width_s, n))`` has the device reduce every replica's samples into the
reference's ``Data.bucket(width_s)`` (instrumentation/data.py:127-158) as they arrive -- count, ``sum()``, ``max()``
per bucket -- instead of recording the samples, and reduces those per sweep cell.  With ``bucket_percentiles=True`` it
also selects every bucket's p50 and p99 from the current bucket's values.  This module holds the host side: the
argument checks, the bucket index restated on the host, the row -> object mapping, the reference's ``BucketedData`` of
one object of one replica, and numpy restatements of the device's cell reductions."""
from __future__ import annotations

import math

import numpy as np

from . import _abi as A
from .instrumentation import BucketedData

MAX_BUCKETS = 1 << 24
MAX_SAMPLE_CAP = 1 << 24
SLICE = 256                 # replicas per first-stage slice of the cell reduction (HS_BUCKET_SLICE)


def check_spec(buckets, end_ns: int) -> tuple[float, int]:
    """``buckets=(width_s, n)`` as ``run_ensemble`` takes it: a finite width > 0 in seconds and 1 <= n <= 2^24
    buckets whose span covers the end time -- every sample up to ``end_ns`` has an index < n (the one event a replica
    processes past the end time may fall beyond; its samples keep their own index)."""
    try:
        w, n = buckets
    except (TypeError, ValueError):
        raise ValueError(f"buckets must be (width_s, n), got {buckets!r}") from None
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)):
        raise ValueError(f"the bucket count must be an int, got {n!r}")
    w, n = float(w), int(n)
    if not (w > 0.0 and math.isfinite(w)):
        raise ValueError(f"the bucket width must be a finite number of seconds > 0, got {w!r}")
    if not 1 <= n <= MAX_BUCKETS:
        raise ValueError(f"the bucket count must be in [1, 2^24], got {n}")
    last = bucket_index(int(end_ns), w)
    if last >= n:
        raise ValueError(f"{n} buckets of {w} s end before the end time {int(end_ns) / 1e9} s (it falls in bucket {last}): "
                         "n * width must exceed the end time")
    return w, n


def check_sample_cap(cap, spec) -> int:
    """``bucket_sample_cap`` of a ``bucket_percentiles=True`` run: an int in [1, 2^24], and buckets to go with it."""
    if spec is None:
        raise ValueError("bucket_percentiles=True needs buckets=(width_s, n)")
    if isinstance(cap, bool) or not isinstance(cap, (int, np.integer)) or not 1 <= int(cap) <= MAX_SAMPLE_CAP:
        raise ValueError(f"bucket_sample_cap must be an int in [1, 2^24], got {cap!r}")
    return int(cap)


def sample_cap_needed(rec) -> int:
    """The sample capacity that holds every bucket of the records ``rec`` (BUCKET_DTYPE): the next power of two at or
    above the largest count."""
    top = max(1, int(rec["count"].max(initial=1)))
    return min(MAX_SAMPLE_CAP, 1 << (top - 1).bit_length())


def bucket_index(ns, w: float):
    """``math.floor(Instant.to_seconds() / w)`` of a time in ns, as ``Data.bucket`` evaluates it: the correctly rounded
    ns / 1e9, then a correctly rounded division by w, then floor (an int for an int, int64 for an array)."""
    if isinstance(ns, (int, np.integer)):
        return math.floor((int(ns) / 1_000_000_000) / w)
    t = np.asarray(ns, dtype=np.int64).astype(np.float64) / 1e9      # exact int64 -> float64 below 2^53 ns (104 days)
    return np.floor(t / w).astype(np.int64)


def rows(model) -> list[int]:
    """The bucketed rows: the model's SINK and PROBE entity ids in entity order (row b = the b-th of them)."""
    k = model.entities["kind"]
    return [i for i in range(len(k)) if int(k[i]) in (A.HS_ENT_SINK, A.HS_ENT_PROBE)]


def row_objects(model, objects) -> list:
    """The object behind each bucketed row: a Sink / LatencyTracker / ThroughputTracker, or for a PROBE row the Probe
    whose ticking (a SOURCE row) targets it."""
    k, tgt = model.entities["kind"], model.entities["target"]
    probe_of = {int(tgt[i]): o for i, o in enumerate(objects) if int(k[i]) == A.HS_ENT_SOURCE and hasattr(o, "data_sink")}
    return [objects[i] if int(k[i]) == A.HS_ENT_SINK else probe_of.get(i) for i in rows(model)]


def read_outputs(eng, spec, cap: int, model, objects, n_cells: int = 1) -> dict:
    """The bucket keys of a bucketed ensemble's output dict, read from the engine ``eng`` after the run's last launch:
    ``buckets`` and ``bucket_past_end`` (the records), ``bucket_totals`` (``n_cells`` cells), ``bucket_width_s``,
    ``bucket_count``, ``bucket_rows`` and ``bucket_objects`` (the rows of ``model``, whose entity ids index
    ``objects``), and with percentiles (``cap`` > 0) ``bucket_percentiles``, ``bucket_percentile_totals`` and
    ``bucket_sample_cap``.  ``Simulation.run_ensemble`` and a linked run's partitions both fill their outputs here."""
    w, nb = spec
    out = {}
    out["buckets"], out["bucket_past_end"] = eng.read_buckets(nb)
    nr = out["buckets"].shape[1]
    out["bucket_totals"] = eng.read_bucket_totals(n_cells, nr, nb)
    out["bucket_width_s"], out["bucket_count"] = w, nb
    out["bucket_rows"] = rows(model)
    out["bucket_objects"] = row_objects(model, objects)
    if cap:
        out["bucket_percentiles"] = eng.read_bucket_percentiles(nb)
        out["bucket_percentile_totals"] = eng.read_bucket_percentile_totals(n_cells, nr, nb)
        out["bucket_sample_cap"] = cap
    return out


def _row_of(out, obj) -> int:
    for b, o in enumerate(out["bucket_objects"]):
        if o is obj or (o is not None and getattr(o, "data_sink", None) is obj):
            return b
    raise KeyError(f"{getattr(obj, 'name', obj)!r} is not a bucketed Sink, tracker or Probe of this run")


def _is_throughput(obj) -> bool:
    """a ThroughputTracker (the mirror's, the reference's, or a subclass of either): its samples are all 1.0"""
    return getattr(obj, "_sample_value", None) == "one" or any(c.__name__ == "ThroughputTracker" for c in type(obj).__mro__)


def replica_sums(rec):
    """sum() of every bucket record: s + c when the compensation is non-zero and finite (hs_neumaier_result)"""
    s, c = rec["sum"], rec["comp"]
    return np.where((c != 0.0) & np.isfinite(c), s + c, s)


def bucketed_data(out, obj, replica: int) -> BucketedData:
    """The reference's ``Data.bucket(width_s)`` of ``obj`` (a Sink, LatencyTracker, ThroughputTracker, Probe or a
    Probe's Data) in replica ``replica`` of a bucketed ``run_ensemble`` result ``out``.  Times, means, counts, maxes
    and sums are those of the replica's complete sample list.  p50 and p99 are those of ``bucket_percentiles=True``
    (NaN for a bucket that overflowed its sample capacity); without it they are NaN (record mode, ``sample_cap``, keeps
    the samples for small runs).  Empty buckets are omitted, as Data.bucket omits them.

    A ThroughputTracker's samples are all 1.0, so its sums, maxes and percentiles are derived here from the counts.
    The device does not know which rows are ThroughputTracker rows: its records, ``out["bucket_percentiles"]``, and
    the per-cell ``out["bucket_totals"]`` / ``out["bucket_percentile_totals"]`` of such a row are over the latencies
    the tracker received, raw device values."""
    b = _row_of(out, obj)
    w, n = out["bucket_width_s"], out["bucket_count"]
    rec = out["buckets"][replica, b]
    keys = [k for k in range(n) if rec["count"][k] > 0]
    idx = keys + ([int(out["bucket_past_end"][replica, b])] if rec["count"][n] > 0 else [])
    slots = keys + ([n] if rec["count"][n] > 0 else [])
    one = _is_throughput(out["bucket_objects"][b])
    sums = replica_sums(rec)
    pct = out["bucket_percentiles"][replica, b] if "bucket_percentiles" in out else None
    res = BucketedData()
    for k, s in zip(idx, slots):
        c = int(rec["count"][s])
        total = float(c) if one else float(sums[s])        # a ThroughputTracker's samples are all 1.0
        res._times.append(k * w)
        res._means.append(total / c)
        res._counts.append(c)
        res._maxes.append(1.0 if one else float(rec["max"][s]))
        res._sums.append(total)
        if pct is None:
            res._p50s.append(math.nan)
            res._p99s.append(math.nan)
        else:                                               # 1.0 * (1 - f) + 1.0 * f rounds to 1.0 for every f
            res._p50s.append(1.0 if one and not math.isnan(pct[s, 0]) else float(pct[s, 0]))
            res._p99s.append(1.0 if one and not math.isnan(pct[s, 1]) else float(pct[s, 1]))
    return res


def _cell_slices(nr: int, n_cells: int, replica_index_base: int, replicas_per_cell: int):
    """The device's slices (hs_read_bucket_totals): (cell, begin, end) for runs of at most 256 consecutive replicas of
    one cell, in index order."""
    cell_of = ((replica_index_base + np.arange(nr)) // replicas_per_cell) % n_cells
    r = 0
    while r < nr:
        c0 = int(cell_of[r])
        end = r + 1
        while end < min(r + SLICE, nr) and cell_of[end] == c0:
            end += 1
        yield c0, r, end
        r = end


def cell_totals_reference(buckets, n_cells: int, *, replica_index_base: int = 0, replicas_per_cell: int = 1):
    """numpy restatement of hs_read_bucket_totals over per-replica records ``buckets`` [replicas, rows, n + 1]
    (BUCKET_DTYPE), in the device's order: slices of at most 256 consecutive replicas of one cell, each folded in
    index order, then each cell's slices in index order.  Returns BUCKET_TOTAL_DTYPE [n_cells, rows, n + 1]."""
    nr = buckets.shape[0]
    shape = buckets.shape[1:]
    out = np.zeros((n_cells,) + shape, A.BUCKET_TOTAL_DTYPE)
    out["max"] = -np.inf
    fields = ("sum", "mean_sum", "mean_sq_sum")
    for c0, r, end in _cell_slices(nr, n_cells, replica_index_base, replicas_per_cell):
        part = {f: np.zeros(shape) for f in fields}
        reps = np.zeros(shape, np.int64); cnt = np.zeros(shape, np.int64); mx = np.full(shape, -np.inf)
        for q in range(r, end):
            rec = buckets[q]
            has = rec["count"] > 0
            s = replica_sums(rec)
            with np.errstate(invalid="ignore", divide="ignore"):
                m = s / rec["count"]
            reps += has; cnt += rec["count"]
            part["sum"] = np.where(has, part["sum"] + s, part["sum"])
            part["mean_sum"] = np.where(has, part["mean_sum"] + m, part["mean_sum"])
            part["mean_sq_sum"] = np.where(has, part["mean_sq_sum"] + m * m, part["mean_sq_sum"])
            mx = np.where(has & (rec["max"] > mx), rec["max"], mx)
        c = out[c0]
        c["replicas"] += reps; c["count"] += cnt
        for f in fields:
            c[f] = c[f] + part[f]
        c["max"] = np.where(mx > c["max"], mx, c["max"])
    return out


def cell_percentile_totals_reference(buckets, pct, n_cells: int, *, replica_index_base: int = 0,
                                     replicas_per_cell: int = 1):
    """numpy restatement of hs_read_bucket_percentile_totals over per-replica records ``buckets`` [replicas, rows, n + 1]
    (BUCKET_DTYPE) and their percentiles ``pct`` [replicas, rows, n + 1, 2], in the device's order and slices (see
    cell_totals_reference); a replica contributes to a bucket only if its record there has samples.  Returns
    BUCKET_PCT_TOTAL_DTYPE [n_cells, rows, n + 1]."""
    shape = buckets.shape[1:]
    out = np.zeros((n_cells,) + shape, A.BUCKET_PCT_TOTAL_DTYPE)
    for c0, r, end in _cell_slices(buckets.shape[0], n_cells, replica_index_base, replicas_per_cell):
        part = {f: np.zeros(shape) for f in A.BUCKET_PCT_TOTAL_DTYPE.names}
        for q in range(r, end):
            has = buckets[q]["count"] > 0
            for f, i in (("p50", 0), ("p99", 1)):
                v = pct[q][..., i]
                part[f + "_sum"] = np.where(has, part[f + "_sum"] + v, part[f + "_sum"])
                part[f + "_sq_sum"] = np.where(has, part[f + "_sq_sum"] + v * v, part[f + "_sq_sum"])
        c = out[c0]
        for f in part:
            c[f] = c[f] + part[f]
    return out
