"""tests/golden/random_fault_models.npz: what the UNMODIFIED reference does on the seeded random models of
tests/random_models.py (random_model and random_model_v2) with their random node-fault schedules
(random_models.random_fault_case), on replica word 0.  Run in the build container (needs /root/reference):

    python tests/golden/gen_random_fault_golden.py

Per model: the summary, the per-entity statistics (the FAULT rows' fired and cancelled counts included), the sketch
states (canonical, random_model) or TTL cache states (random_model_v2) and the summary's events_cancelled."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import gen_fault_golden as GF                 # noqa: E402
from random_models import FAULT_SEEDS_V1, FAULT_SEEDS_V2    # noqa: E402
from test_faults import reference_case_kw     # noqa: E402

out = {}
for version, seeds in ((1, FAULT_SEEDS_V1), (2, FAULT_SEEDS_V2)):
    for seed in seeds:
        model, build, kw, plan, cancel = reference_case_kw(version, seed, 0)
        fm, ref, meta = GF.run_case(model, build, kw)
        p = f"v{version}s{seed}_"
        out[p + "summary"] = ref["summaries"]
        out[p + "stats"] = ref["entity_stats"]
        if "sketches" not in ref:
            out[p + "sketches"] = np.zeros(0, np.uint8)
        else:
            out[p + "sketches"] = fm.canonical_sketches(ref["sketches"])[0] if version == 1 else ref["sketches"]
        out[p + "cancelled"] = meta["events_cancelled"]
        print(f"v{version} seed {seed}: {len(plan)} faults, cancelled {int(meta['events_cancelled'])} ->",
              int(ref["summaries"]["events_processed"][0]), "events")
out["seeds_v1"] = np.array(FAULT_SEEDS_V1)
out["seeds_v2"] = np.array(FAULT_SEEDS_V2)
np.savez_compressed(os.path.join(HERE, "random_fault_models.npz"), **out)
print("wrote random_fault_models.npz for", len(FAULT_SEEDS_V1), "+", len(FAULT_SEEDS_V2), "seeds")
