"""tests/golden/size_<name>.npz: what the UNMODIFIED reference does on the large models of tests/model_size_lib.py
(fixture_models): the 512- and 1 024-server farms (round robin, and BASELINE configs[3]'s consistent-hash key table),
a server with about 35 000 requests in service, and a load balancer over 65 531 Counters with a Probe (65 535 rows).
Replica word 0, short horizons.  Each fixture keeps the summary, the entity statistics, the last FIXTURE_TAIL event
records and Sink samples, and the counts; the order hash covers every event.  Run in the build container (needs the
reference checkout):

    python tests/golden/gen_model_size_golden.py [name ...]      # all fixtures, or the named ones
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import ref_harness as RH                      # noqa: E402
from model_size_lib import FIXTURE_SEED, FIXTURE_TAIL, fixture_models   # noqa: E402

for name, (model, end_ns, kw) in fixture_models().items():
    if sys.argv[1:] and name not in sys.argv[1:]:
        continue
    ref = RH.run_reference(model, seed=FIXTURE_SEED, rid=0, end_ns=end_ns, **kw)
    s = ref["summaries"]
    np.savez_compressed(os.path.join(HERE, f"size_{name}.npz"), summaries=s, entity_stats=ref["entity_stats"],
                        records_tail=ref["records"][-FIXTURE_TAIL:], samples_tail=ref["sink_samples"][-FIXTURE_TAIL:],
                        meta=np.array([FIXTURE_SEED, end_ns], np.int64))
    print(name, "->", int(s["events_processed"][0]), "events,", int(s["heap_left"][0]), "pending at the end")
