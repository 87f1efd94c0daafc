"""The oracle's multi-replica trace entry point (hs_oracle_run_trace) against the stock-seeded reference.

tests/golden/stockens_*.npz hold eight runs of the UNMODIFIED reference per model family, seeded random.seed(s);
numpy.random.seed(s) for eight consecutive seeds.  One oracle call with one row of draws per replica -- the rows
happysim_b200.api.stock_streams builds for an rng="stock" ensemble -- must reproduce every one of them bit for bit."""
import numpy as np
import pytest

import golden_lib as G
import oracle_lib as O
from happysim_b200 import _abi as A
from happysim_b200.api import stock_streams


def _uses(model):
    """(has a Poisson source, has an exponential server): the streams the family draws from"""
    e = model.entities
    src, srv = e["kind"] == A.HS_ENT_SOURCE, e["kind"] == A.HS_ENT_SERVER
    return bool((e["i0"][src] == A.HS_ARR_POISSON).any()), bool((e["i2"][srv] == A.HS_SVC_EXPONENTIAL).any())


@pytest.mark.parametrize("name", G.case_names("stockens_"))
def test_oracle_reproduces_every_seed_of_a_stock_ensemble(name):
    model, kw, z = G.load(name)
    n, n_draws = len(z["summaries"]), int(z["n_draws"])
    arr, svc = stock_streams(kw["seed"], n, n_draws)
    got = O.oracle_run_trace(model, O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n,
                                                  **G.stock_ensemble_caps(z)), arr, svc)
    for k in range(n):
        G.check_stock_ensemble(z, k, got, k)
    # every replica stayed inside its rows, and a stream the family draws from is drawn a few hundred times
    assert got["arr_used"].max() <= n_draws and got["svc_used"].max() <= n_draws
    poisson, expo = _uses(model)
    assert (got["arr_used"].min() >= 200) if poisson else not got["arr_used"].any()
    assert (got["svc_used"].min() >= 200) if expo else not got["svc_used"].any()


@pytest.mark.parametrize("name", G.case_names("stock_"))
def test_single_replica_stock_fixture_is_one_row_of_many(name):
    """A stock_<case>.npz run placed at slot 2 of five replicas whose other rows hold other seeds' draws: the slot
    reads its own row."""
    model, kw, z = G.load(name)
    n = len(z["trace_targets"])
    arr, svc = stock_streams(kw["seed"] + 1000, 5, n)
    arr[2], svc[2] = z["trace_targets"], z["trace_service"]
    got = O.oracle_run_trace(model, O.make_params(n_replicas=5, end_ns=kw["end_ns"], **G.caps(z)), arr, svc)
    G.check_against(z, got, r=2)
    assert int(got["arr_used"][2]) <= n and int(got["svc_used"][2]) <= n
    for r in (0, 1, 3, 4):
        assert got["summaries"][r]["order_hash"] != got["summaries"][2]["order_hash"]


def test_stream_without_draws_comes_from_philox():
    """A stream given no draws (zero columns, or None) comes from Philox, as after Engine.set_trace with an empty row:
    service start k takes Philox draw k whatever the arrivals, so the service times equal those of a Philox run."""
    model, kw, z = G.load("stock_mm1_seed42")
    p = O.make_params(seed=5, end_ns=kw["end_ns"], n_replicas=3, record_cap=0, sample_cap=0, service_cap=8192)
    arr, _ = stock_streams(42, 3, len(z["trace_targets"]))
    philox = O.oracle_run(model, p)
    for none in (np.zeros((3, 0)), None):
        mixed = O.oracle_run_trace(model, p, arr, none)
        assert not mixed["svc_used"].any() and (mixed["arr_used"] > 200).all()
        for r in range(3):
            k = int(min(mixed["summaries"]["n_service_samples"][r], philox["summaries"]["n_service_samples"][r]))
            assert k > 200 and mixed["service_samples"][r][:k].tobytes() == philox["service_samples"][r][:k].tobytes()
            assert mixed["summaries"][r]["order_hash"] != philox["summaries"][r]["order_hash"]
