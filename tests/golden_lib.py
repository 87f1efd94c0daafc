"""Load the committed reference fixtures (tests/golden/*.npz)."""
import glob
import os
import sys

import numpy as np

import happysim_b200 as hs

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# The unmodified reference (its package and examples) as build() installs it from the reference checkout
# (oracle/Makefile, target `ref`); tests that need the reference's own classes import it from here.
REF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
HAVE_REF = os.path.isdir(os.path.join(REF_DIR, "happysimulator"))
NO_REF = "the reference is not installed in oracle/_ref (build() installs it when the reference checkout is present)"


def import_reference():
    """Put oracle/_ref on sys.path and return the reference's happysimulator package."""
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)
    import happysimulator
    return happysimulator


def case_names(prefix):
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, prefix + "*.npz")))


def load(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    model = hs.FlatModel(entities=z["entities"], names=[str(s) for s in z["names"]], backends=z["backends"],
                         key_table=z["key_table"])
    if "profiles" in z.files and len(z["profiles"]):
        model.profiles = z["profiles"]
    if "profile_table" in z.files and len(z["profile_table"]):
        model.profile_table = z["profile_table"]
    if "sketch_tables" in z.files and len(z["sketch_tables"]):
        model.sketch_tables = z["sketch_tables"]
    if "key_cdf" in z.files and len(z["key_cdf"]):
        model.key_cdf = z["key_cdf"]
    seed, rid, end_ns = (int(v) for v in z["meta"])
    return model, dict(seed=seed, rid_base=rid, end_ns=end_ns), z


def caps(z):
    """Ring capacities that retain the whole run, so the fixture's prefix can be compared."""
    return dict(record_cap=int(z["n_records"]) + 1, sample_cap=int(z["n_samples"]) + 1,
                service_cap=int(z["n_service"]) + 1)


def check_against(z, got, r=0):
    """Compare replica ``r`` of an oracle/engine result with a reference fixture."""
    s, ws = got["summaries"][r], z["summaries"][0]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (f, int(s[f]), int(ws[f]))
    assert got["entity_stats"][r].tobytes() == z["entity_stats"][0].tobytes(), "entity statistics differ"
    n = len(z["records"])
    assert got["records"][r][:n].tobytes() == z["records"].tobytes(), "event records differ"
    n = len(z["sink_samples"])
    if n:
        assert got["sink_samples"][r][:n].tobytes() == z["sink_samples"].tobytes(), "sink samples differ"
    n = len(z["service_samples"])
    if n:
        assert got["service_samples"][r][:n].tobytes() == z["service_samples"].tobytes(), "service samples differ"
    if "sketch_state" in z.files and len(z["sketch_state"]):
        model = load(str(z["case_name"]))[0] if "case_name" in z.files else None
        a, b = got["sketches"][r], z["sketch_state"]
        if model is not None:        # TDigest rows carry dead slots (leftovers of merges): compare the live state
            a, b = model.canonical_sketches(a)[0], model.canonical_sketches(b)[0]
        assert a.tobytes() == b.tobytes(), "sketch registers / counters differ"


def load_linked(name):
    """A linked-partition fixture (tests/golden/gen_linked_golden.py): (LinkedModel, dict(seed, end_ns), npz)."""
    from happysim_b200.linked import LinkedModel, LinkSpec
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    names = [str(s) for s in z["names"]]
    models, links = [], []
    for q in range(len(names)):
        pre = f"p{q}_"
        m = hs.FlatModel(entities=z[pre + "entities"], names=[str(s) for s in z[pre + "enames"]],
                         backends=z[pre + "backends"], key_table=z[pre + "key_table"])
        m.outbox_cap, m.inbox_cap = (int(v) for v in z[pre + "caps"])
        models.append(m)
        links.append([LinkSpec(int(a[0]), int(a[1]), float(b[0]), float(b[1]), int(a[2]))
                      for a, b in zip(z[pre + "links"], z[pre + "link_params"])])
    lm = LinkedModel(models, names, links, window_s=float(z["window_s"]), n_streams=int(z["n_streams"]))
    seed, end_ns = (int(v) for v in z["meta"])
    return lm, dict(seed=seed, end_ns=end_ns), z


def linked_caps(z, q):
    pre = f"p{q}_"
    return dict(record_cap=len(z[pre + "records"]) + 1, sample_cap=len(z[pre + "sink_samples"]) + 1,
                service_cap=len(z[pre + "service_samples"]) + 1)


def check_linked_partition(z, q, got, r=0):
    """Partition q of a linked fixture against replica r of an oracle / engine result."""
    pre = f"p{q}_"
    s, ws = got["summaries"][r], z[pre + "summaries"][0]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (q, f, int(s[f]), int(ws[f]))
    assert int(s["status"]) == 0
    assert got["entity_stats"][r].tobytes() == z[pre + "entity_stats"][0].tobytes(), f"partition {q}: entity statistics differ"
    n = len(z[pre + "records"])
    assert got["records"][r][:n].tobytes() == z[pre + "records"].tobytes(), f"partition {q}: event records differ"
    n = len(z[pre + "sink_samples"])
    if n:
        assert got["sink_samples"][r][:n].tobytes() == z[pre + "sink_samples"].tobytes(), f"partition {q}: sink samples differ"
    n = len(z[pre + "service_samples"])
    if n:
        assert got["service_samples"][r][:n].tobytes() == z[pre + "service_samples"].tobytes(), f"partition {q}: service samples differ"
    if pre + "sketch_state" in z.files and len(z[pre + "sketch_state"]):
        assert got["sketches"][r].tobytes() == z[pre + "sketch_state"].tobytes(), f"partition {q}: sketch state differs"


def stock_ensemble_caps(z):
    """Ring capacities that retain the whole run of every replica of a stock-ensemble fixture."""
    return dict(record_cap=int(z["n_records"].max()) + 1, sample_cap=int(z["n_samples"].max()) + 1,
                service_cap=int(z["n_service"].max()) + 1)


def check_stock_ensemble(z, k, got, r):
    """Replica k of a stock-ensemble fixture (tests/golden/gen_stock_ensemble_golden.py) against replica r of an oracle /
    engine result whose rings retain the whole run (stock_ensemble_caps)."""
    s, ws = got["summaries"][r], z["summaries"][k]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (k, f, int(s[f]), int(ws[f]))
    assert got["entity_stats"][r].tobytes() == z["entity_stats"][k].tobytes(), f"seed {k}: entity statistics differ"
    n = min(int(z["n_records"][k]), z["records"].shape[1])
    assert got["records"][r][:n].tobytes() == z["records"][k][:n].tobytes(), f"seed {k}: event records differ"
    n = int(z["n_samples"][k])
    assert got["sink_samples"][r][:n].tobytes() == z["sink_samples"][k][:n].tobytes(), f"seed {k}: sink samples differ"
    n = int(z["n_service"][k])
    assert got["service_samples"][r][:n].tobytes() == z["service_samples"][k][:n].tobytes(), f"seed {k}: service times differ"
