"""tests/golden/prio_*.npz and tests/golden/prio_random_models.npz: what the UNMODIFIED reference does on the models
of tests/priority_models.py, with the reference's own PriorityQueue(capacity, key=happysim_b200.PriorityByKey(values))
in front of its own Server.  Run in the build container (needs the reference checkout):

    python tests/golden/gen_priority_golden.py

ref_harness builds the reference's object graph with the Philox plug-ins (a PRIORITY row first gets a FIFOQueue of
the row's capacity); the Server's queue policy is then replaced by the PriorityQueue, before the Simulation exists.
prio_<name>.npz: the event records, Sink samples, service times, entity statistics and summary of replica word 0 (the
format of gen_golden.save_case).  prio_random_models.npz: summary and entity statistics per random seed."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import ref_harness as RH                      # noqa: E402
from gen_golden import save_case             # noqa: E402
import priority_models as PM                 # noqa: E402
import happysim_b200 as hs                   # noqa: E402

SEED = 20261018


def run_reference_priority(model, extras, *, seed, end_s):
    RH._import_reference()
    from happysimulator.components.queue_policy import PriorityQueue
    from happysimulator.core.simulation import Simulation
    from happysimulator.core.temporal import Instant
    ctx = RH.run_reference(model, seed=seed, rid=0, end_ns=int(end_s * 1e9), zipf_s=extras["zipf_s"], _build_only=True)
    for i, values in extras["priorities"].items():
        srv = ctx["objs"][i]
        cap = int(model.entities["l0"][i])
        srv.queue.policy = PriorityQueue(capacity=cap if cap >= 0 else float("inf"), key=hs.PriorityByKey(values))
    sim = Simulation(end_time=Instant(int(end_s * 1e9)), sources=ctx["sources"], entities=ctx["entities"],
                     probes=ctx["probes"] or None)
    recs = ctx["attach"](sim)
    summary = sim.run()
    for i, values in extras["priorities"].items():          # the policy the run used, as the device publishes it
        pol = ctx["objs"][i].queue.policy
        assert pol._insert_counter == ctx["objs"][i].stats_accepted
    return ctx["extract"](sim, recs, summary)


def main():
    for name, (model, end_s, extras) in PM.fixture_models().items():
        ref = run_reference_priority(model, extras, seed=SEED, end_s=end_s)
        save_case(os.path.join(HERE, f"prio_{name}.npz"), model, ref, dict(seed=SEED, rid=0, end_s=end_s))
        print(f"prio_{name}: {len(ref['records'])} events, dropped",
              [int(ref["entity_stats"][0][i]["c1"]) for i in extras["priorities"]])
    out = {}
    for s in PM.RANDOM_SEEDS:
        model, end_s, extras = PM.random_priority_model(s)
        ref = run_reference_priority(model, extras, seed=SEED + s, end_s=end_s)
        out[f"s{s}_summary"], out[f"s{s}_stats"] = ref["summaries"], ref["entity_stats"]
        print(f"random seed {s}: {int(ref['summaries']['events_processed'][0])} events")
    out["seeds"] = np.array(PM.RANDOM_SEEDS)
    out["base_seed"] = np.int64(SEED)
    np.savez_compressed(os.path.join(HERE, "prio_random_models.npz"), **out)


if __name__ == "__main__":
    main()
