"""``happysim_b200.install()`` -- route the REFERENCE's own entry points through the CUDA engine.

After ``install()`` an unchanged reference script (``from happysimulator import Simulation, Source, ...``) runs
its ``Simulation(...).run()`` on the device whenever its object graph lowers (lowering.py) and falls through to the
reference's Python loop, untouched, when it does not (user-defined entities, auto-termination, tracing, the debugger
control surface, a start time other than the epoch, faults other than CrashNode / PauseNode): nothing is ever
mis-simulated.  A fault schedule of node faults lowers to FAULT rows: the crash flag and its drop run on the device.

What is patched (reference paths under happysimulator/):
  core/simulation.py:66   Simulation.__init__   wrapped only to snapshot numpy's global generator BEFORE the
                                                sources draw their first arrival (source.start, :145-154)
  core/simulation.py:230  Simulation.run        lower -> hs_run -> write the results back onto the script's own
                                                entity objects (sink.latencies_s, server.stats, ...), return the
                                                reference's own SimulationSummary type
  parallel/runner.py:115  ParallelRunner.run_replicas   the replicas as ONE device ensemble (Philox key base_seed + i)

Randomness.  ``Simulation.run`` is reproduced DRAW FOR DRAW: the engine's stock-generator mode (hs_set_trace)
consumes exactly the variates the reference would have taken from its two process-global MT19937 streams --
numpy's (Poisson arrivals, load/providers/poisson_arrival.py:31) from the state snapshotted at construction,
Python's ``random`` (service times, distributions/exponential.py:43) from its state when run() is called -- so a
script seeded with ``random.seed(s); numpy.random.seed(s)`` prints the same numbers with and without
``install()``; afterwards both global generators are advanced by the number of draws the run consumed.
``run_replicas`` uses the Philox streams keyed by ``base_seed + i`` (the reference's worker processes inherit
numpy's state by fork and all share one arrival stream unless build_fn reseeds it -- not a behaviour to mirror).
"""
from __future__ import annotations

import math
import time as _time

import numpy as np

from . import _abi as A
from . import api, lowering

_state = {"installed": False, "orig": {}, "stats": {"device_runs": 0, "fallbacks": 0, "last_fallback_reason": None},
          "device": 0, "verbose": False}


def stats() -> dict:
    """Counters since install(): how many run() calls went to the device, how many fell through and why."""
    return dict(_state["stats"])


def _eligible(sim):
    """None if the reference Simulation can run on the device as it stands, else the reason it cannot."""
    import happysimulator.core.temporal as T
    if sim._end_time == T.Instant.Infinity:
        return "auto-termination (no end_time / duration)"
    if int(sim._start_time.nanoseconds) != 0:
        return "start_time other than Instant.Epoch"
    if sim._tracing_enabled:
        return "trace_recorder"
    if sim._control is not None or sim._is_running or sim._event_router is not None or sim._pre_run_event_specs:
        return "control surface / re-entrant run / partition router / scheduled pre-run events"
    return None


def _trace_fn_from_states(np_state, py_state):
    """n_draws -> (arrival targets, service variates) exactly as the reference would draw them from the two global
    generators in the given states (api.stock_streams does the same from a seed)."""
    import random as _random

    def fn(n_draws: int):
        rs = np.random.RandomState()
        rs.set_state(np_state)
        u = rs.random_sample(n_draws)
        arr = np.array([[-math.log(1.0 - x) for x in u]], np.float64)
        rnd = _random.Random()
        rnd.setstate(py_state)
        svc = np.array([[-math.log(1.0 - rnd.random()) for _ in range(n_draws)]], np.float64)
        return arr, svc
    return fn


def install(*, device: int = 0, verbose: bool = False) -> None:
    """Patch the importable reference package (idempotent).  Raises ImportError if ``happysimulator`` is missing."""
    import random as _random
    import happysimulator.core.simulation as S
    import happysimulator.parallel.runner as R
    from happysimulator.instrumentation.summary import EntitySummary, QueueStats, SimulationSummary

    _state["device"], _state["verbose"] = device, verbose
    if _state["installed"]:
        return
    orig_init, orig_run, orig_replicas = S.Simulation.__init__, S.Simulation.run, R.ParallelRunner.run_replicas
    _state["orig"] = {"init": orig_init, "run": orig_run, "run_replicas": orig_replicas}

    def __init__(self, *a, **kw):
        self._hs_np_state = np.random.get_state()          # before source.start() draws the first arrivals
        orig_init(self, *a, **kw)

    def _to_ref_summary(sm):
        ents = {k: EntitySummary(name=v.name, entity_type=v.entity_type, events_handled=v.events_handled,
                                 queue_stats=None if v.queue_stats is None else QueueStats(
                                     peak_depth=v.queue_stats.peak_depth, total_accepted=v.queue_stats.total_accepted,
                                     total_dropped=v.queue_stats.total_dropped))
                for k, v in sm.entities.items()}
        return SimulationSummary(duration_s=sm.duration_s, total_events_processed=sm.total_events_processed,
                                 events_cancelled=sm.events_cancelled, events_per_second=sm.events_per_second,
                                 wall_clock_seconds=sm.wall_clock_seconds, entities=ents)

    def run(self):
        st = _state["stats"]
        why = _eligible(self)
        model = objects = None
        if why is None:
            try:
                model, objects = lowering.lower(self._sources, self._entities, probes=self._probes or None,
                                                horizon_s=float(int(self._end_time.nanoseconds)) / 1e9,
                                                fault_schedule=self._fault_schedule)
            except lowering.UnsupportedModelError as e:
                why = str(e)
        if why is not None:
            st["fallbacks"] += 1
            st["last_fallback_reason"] = why
            if _state["verbose"]:
                print(f"[happysim_b200] {type(self).__name__}.run: reference loop ({why})")
            return orig_run(self)
        np_state = getattr(self, "_hs_np_state", None) or np.random.get_state()
        py_state = _random.getstate()
        t0 = _time.monotonic()
        sm = api.run_lowered(self, model, objects, device=_state["device"], trace_fn=_trace_fn_from_states(np_state, py_state))
        # leave both global generators where a reference run would have left them
        kinds = model.entities["kind"]
        n_arr = sum(int(getattr(o, "_generated_count", 0)) + 1 for i, o in enumerate(objects)
                    if int(kinds[i]) == A.HS_ENT_SOURCE and int(model.entities["i0"][i]) == A.HS_ARR_POISSON)
        n_svc = sum(len(getattr(o, "_service_times", ())) for i, o in enumerate(objects)
                    if int(kinds[i]) == A.HS_ENT_SERVER and int(model.entities["i2"][i]) == A.HS_SVC_EXPONENTIAL)
        rs = np.random.RandomState()
        rs.set_state(np_state)
        if n_arr:
            rs.random_sample(n_arr)
        np.random.set_state(rs.get_state())
        for _ in range(n_svc):
            _random.random()
        self._summary = _to_ref_summary(sm)
        self._events_processed = sm.total_events_processed
        self._current_time = type(self._start_time)(int(round(sm.duration_s * 1e9)))
        st["device_runs"] += 1
        if _state["verbose"]:
            print(f"[happysim_b200] {type(self).__name__}.run: {sm.total_events_processed} events on cuda:{_state['device']} "
                  f"in {_time.monotonic() - t0:.3f} s")
        return self._summary

    def run_replicas(self, build_fn, n_replicas, base_seed=42):
        st = _state["stats"]
        try:
            _random.seed(base_seed)
            ref_sim = build_fn()
            why = _eligible(ref_sim)
            if why is not None:
                raise lowering.UnsupportedModelError(why)
            model, objects = lowering.lower(ref_sim._sources, ref_sim._entities, probes=ref_sim._probes or None,
                                            horizon_s=float(int(ref_sim._end_time.nanoseconds)) / 1e9,
                                            fault_schedule=ref_sim._fault_schedule)
        except lowering.UnsupportedModelError as e:
            st["fallbacks"] += 1
            st["last_fallback_reason"] = str(e)
            return orig_replicas(self, build_fn, n_replicas, base_seed)
        sim = api.Simulation._from_lowered(model, objects, sources=ref_sim._sources, entities=ref_sim._entities,
                                           end_ns=ref_sim._end_time.nanoseconds, seed=base_seed, device=_state["device"],
                                           instant_cls=type(ref_sim._start_time))
        res = api.ParallelRunner().run_replicas(lambda: sim, n_replicas, base_seed, flags=0)
        st["device_runs"] += 1
        return [R.ParallelResult(name=r.name, summary=_to_ref_summary(r.summary)) for r in res]

    S.Simulation.__init__ = __init__
    S.Simulation.run = run
    R.ParallelRunner.run_replicas = run_replicas
    _state["installed"] = True


def uninstall() -> None:
    """Restore the reference's own methods."""
    if not _state["installed"]:
        return
    import happysimulator.core.simulation as S
    import happysimulator.parallel.runner as R
    S.Simulation.__init__ = _state["orig"]["init"]
    S.Simulation.run = _state["orig"]["run"]
    R.ParallelRunner.run_replicas = _state["orig"]["run_replicas"]
    _state["installed"] = False
