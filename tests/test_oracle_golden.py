"""The CPU oracle against the fixtures recorded from the UNMODIFIED reference.

philox_*: the reference was driven through its own plug-in points by the shared
Philox sampler (tests/golden/gen_golden.py); the oracle must reproduce the whole
processed-event sequence (hash over every event), counts, statistics bit for bit.
stock_*:  the reference ran with its stock MT19937 streams (random.seed(42);
np.random.seed(42): the README quick-start known answers, SURVEY.md 8(c)); the
oracle is fed the generators' outputs and must land on the same answers."""
import numpy as np
import pytest

import golden_lib as G
import oracle_lib as O


@pytest.mark.parametrize("name", G.case_names("philox_"))
def test_oracle_reproduces_reference_with_philox_plugins(name):
    model, kw, z = G.load(name)
    got = O.oracle_run(model, O.make_params(**G.caps(z), **kw))
    G.check_against(z, got)


@pytest.mark.parametrize("name", G.case_names("stock_"))
def test_oracle_reproduces_stock_seed_run_from_its_rng_outputs(name):
    model, kw, z = G.load(name)
    kw.pop("seed"), kw.pop("rid_base")
    got = O.oracle_run_trace(model, O.make_params(**G.caps(z), **kw),
                             z["trace_targets"], z["trace_service"])
    G.check_against(z, got)


def test_readme_quickstart_known_answers():
    """SURVEY.md 8(c): random.seed(42); np.random.seed(42); M/M/1 rate 8, mean 0.1 s, 60 s."""
    model, kw, z = G.load("stock_mm1_seed42")
    assert int(z["summaries"]["events_processed"][0]) == 3621
    assert int(z["summaries"]["final_time_ns"][0]) == 60038804895
    assert int(z["summaries"]["heap_left"][0]) == 2
    st = z["entity_stats"][0]
    assert int(st[0]["c0"]) == 483 and int(st[1]["c2"]) == 482 and int(st[2]["c0"]) == 482
    assert float(st[2]["f0"]) / 482 == 0.5696996189709543
    first = [(int(r["time_ns"]), int(r["sort_index"]), int(r["kind"])) for r in z["records"][:10]]
    assert first == [(58658511, 0, 0), (58658511, 0, 2), (58658511, 2, 3), (58658511, 3, 4), (58658511, 4, 5),
                     (58658511, 0, 6), (160664539, 6, 7), (160664539, 7, 8), (160664539, 8, 4), (434923689, 1, 0)]


def test_reference_counter_kat():
    """tests/integration/core_simulation/test_simulation_basic_counter.py:7-34 of the reference:
    constant source at 1/s into a Counter for 60 s -> 61 ticks generated, 60 counted."""
    model, kw, z = G.load("philox_source_to_counter")
    got = O.oracle_run(model, O.make_params(**kw))
    st = got["entity_stats"][0]
    assert int(st[0]["c0"]) == 61 and int(st[1]["c0"]) == 60


def test_order_hash_off_is_zero_even_before_the_first_event():
    """With HS_RUN_ORDER_HASH off every engine reports order_hash 0; so must the oracle for a replica paused before
    it has processed any event (its hash never left HS_HASH_INIT)."""
    import happysim_b200 as hs
    s = O.oracle_run(hs.mm1(rate=0.5), O.make_params(seed=3, end_ns=10**10, window_end_ns=10**9, n_replicas=64,
                                                      flags=0))["summaries"]
    assert (s["events_processed"] == 0).any() and (s["events_processed"] > 0).any()
    assert (s["order_hash"] == 0).all()
