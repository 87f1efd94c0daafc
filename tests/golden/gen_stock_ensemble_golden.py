"""Generate tests/golden/stockens_<family>.npz from the UNMODIFIED reference with its STOCK generators.

    python tests/golden/gen_stock_ensemble_golden.py [family-substring]     # needs the reference checkout

For every family of tests/stock_ensemble_models.py the reference runs once per seed s = s0 .. s0 + 7, seeded
``random.seed(s); numpy.random.seed(s)`` (ref_harness.run_reference(..., stock_rng=True)): row s - s0 of
``happysim_b200.api.stock_streams(s0, 8, n, 1)`` holds exactly the draws that run took from the two streams.  The
model stored is what ``Simulation`` lowers the family to, so the oracle, the engines and ``ParallelRunner.run_sweep``
all run the same rows.

Per replica k the file holds what golden_lib.check_against compares for one replica: the summary (order hash over
the whole run), the entity statistics, the first MAX_REC event records, and the Sink and service-time samples --
all of them, zero-padded to the longest replica (n_records / n_samples / n_service give the real counts).
``n_draws`` is a row length that covers every replica's draws of both streams.

The files are named stockens_*, not stock_*: the single-run fixtures' tests list every stock_*.npz and expect a
single replica with its trace stored in the file.

All eight families can be expressed in stock mode; none is dropped."""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import ref_harness as RH  # noqa: E402
import stock_ensemble_models as SM  # noqa: E402
from happysim_b200 import _abi as A  # noqa: E402

MAX_REC = 256


def padded(rows, dtype):
    out = np.zeros((len(rows), max(1, max(len(r) for r in rows))), dtype)
    for k, r in enumerate(rows):
        out[k, :len(r)] = r
    return out


def generate(name):
    _, s0, end_s, _ = SM.FAMILIES[name]
    model = SM.simulation(name).model
    end_ns = int(round(end_s * 1e9))
    refs = [RH.run_reference(model, seed=s0 + k, end_ns=end_ns, stock_rng=True) for k in range(SM.N_SEEDS)]
    recs = [r["records"] for r in refs]
    np.savez_compressed(
        os.path.join(HERE, f"stockens_{name}.npz"),
        entities=model.entities, backends=model.backends, key_table=model.key_table, profiles=model.profiles,
        profile_table=model.profile_table, names=np.array(model.names),
        meta=np.array([s0, 0, end_ns], dtype=np.int64),
        summaries=np.concatenate([r["summaries"] for r in refs]),
        entity_stats=np.concatenate([r["entity_stats"] for r in refs]),
        n_records=np.array([len(r) for r in recs], np.int64), records=padded([r[:MAX_REC] for r in recs], A.RECORD_DTYPE),
        n_samples=np.array([len(r["sink_samples"]) for r in refs], np.int64),
        sink_samples=padded([r["sink_samples"] for r in refs], A.SAMPLE_DTYPE),
        n_service=np.array([len(r["service_samples"]) for r in refs], np.int64),
        service_samples=padded([r["service_samples"] for r in refs], np.float64),
        # every processed event takes at most one draw: the longest run bounds both streams
        n_draws=np.int64(max(len(r) for r in recs)),
        case_name=np.array(f"stockens_{name}"),
    )
    ev = [int(r["summaries"]["events_processed"][0]) for r in refs]
    print(f"stockens_{name}: seeds {s0}..{s0 + SM.N_SEEDS - 1}, events {min(ev)}..{max(ev)}")


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    for name in SM.FAMILIES:
        if only in name:
            generate(name)


if __name__ == "__main__":
    main()
