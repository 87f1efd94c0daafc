"""tests/golden/sweep_cells.npz: what the UNMODIFIED reference does on each configuration of two sweeps whose
configurations run as the cells of one launch (tests/sweep_models.py): a CachingServer farm at four TTLs and a
load-balanced farm into a QuantileEstimator at three compressions of one buffer size int(2c).  Configuration c runs
with replica word c, as cell c of a launch with one replica per cell does.  Run in the build container (needs the
reference checkout):

    python tests/golden/gen_sweep_cells_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import ref_harness as RH                      # noqa: E402
from sweep_models import FIXTURE_END_NS, FIXTURE_SEED, fixture_models   # noqa: E402

out = {}
for name, (model, plains) in fixture_models().items():
    for c, m in enumerate(plains):
        ref = RH.run_reference(m, seed=FIXTURE_SEED, rid=c, end_ns=FIXTURE_END_NS)
        out[f"{name}_c{c}_summary"] = ref["summaries"]
        out[f"{name}_c{c}_stats"] = ref["entity_stats"]
        out[f"{name}_c{c}_sketches"] = ref["sketches"] if "sketches" in ref else np.zeros(0, np.uint8)
        print(name, c, "->", int(ref["summaries"]["events_processed"][0]), "events")
np.savez_compressed(os.path.join(HERE, "sweep_cells.npz"), **out)
print("wrote sweep_cells.npz")
