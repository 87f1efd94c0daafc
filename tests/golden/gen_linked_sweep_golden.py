"""Fixture for linked runs whose replicas are sweep cells: the unmodified reference's ParallelSimulation +
WindowedCoordinator (ref_harness.run_reference_linked) run once per configuration, for configurations of one linked
topology that differ in link latency and packet loss.

    python tests/golden/gen_linked_sweep_golden.py        # needs the reference; writes tests/golden/lsweep_cells.npz

Cases: the tandem over a constant-latency link (gen_linked_golden.tandem_over_a_link) and the lossy fan-out whose two
exponential links share one latency object (gen_linked_golden.lossy_fanout), four configurations each; one of the
fan-out's configurations loses nothing.  Per case: the partition models and links of configuration 0, the per-cell link
table, and per configuration and partition the reference's summaries, entity statistics, event records, Sink samples,
service times and sketch state, and the coordinator's cross-partition event count."""
import dataclasses
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import conftest  # noqa: F401,E402
import gen_linked_golden as GL  # noqa: E402
import ref_harness as RH  # noqa: E402

# per case: (LinkedModel, seed, end_s, per configuration the (latency mean s, packet loss) of every link, partition by partition)
CASES = {
    "tandem": (GL.tandem_over_a_link, 5, 4.0,
               [[[(0.05, 0.0)], []], [[(0.08, 0.1)], []], [[(0.12, 0.0)], []], [[(0.05, 0.3)], []]]),
    "fanout": (GL.lossy_fanout, 11, 3.0,
               [[[(0.04, 0.15), (0.04, 0.3)], [(0.025, 0.0)], []],
                [[(0.06, 0.0), (0.06, 0.0)], [(0.025, 0.0)], []],
                [[(0.03, 0.25), (0.03, 0.05)], [(0.05, 0.1)], []],
                [[(0.1, 0.15), (0.1, 0.3)], [(0.03, 0.0)], []]]),
}


def configured(lm, cell):
    """``lm`` with the link parameters of one configuration"""
    links = [[dataclasses.replace(l, latency_mean_s=m, packet_loss=p) for l, (m, p) in zip(ls, cs)] for ls, cs in zip(lm.links, cell)]
    return dataclasses.replace(lm, links=links)


def main():
    z = {}
    for name, (make, seed, end_s, cells) in CASES.items():
        lm = make()
        pre = f"{name}_"
        z[pre + "names"] = np.array(lm.names)
        z[pre + "window_s"], z[pre + "n_streams"] = np.float64(lm.window_s), np.int64(lm.n_streams)
        z[pre + "meta"] = np.array([seed, int(end_s * 1e9), len(cells)], dtype=np.int64)
        for q, m in enumerate(lm.models):
            pq = f"{pre}p{q}_"
            z[pq + "entities"], z[pq + "backends"], z[pq + "key_table"] = m.entities, m.backends, m.key_table
            z[pq + "enames"] = np.array(m.names)
            z[pq + "caps"] = np.array([m.outbox_cap, m.inbox_cap], dtype=np.int64)
            z[pq + "links"] = np.array([[l.dest, l.latency_kind, l.stream] for l in lm.links[q]], dtype=np.int64).reshape(-1, 3)
            z[pq + "cell_links"] = np.array([c[q] for c in cells], dtype=np.float64).reshape(len(cells), len(lm.links[q]), 2)
        for c, cell in enumerate(cells):
            lc = configured(lm, cell)
            lc.validate()
            outs, summ = RH.run_reference_linked(lc, seed=seed, end_ns=int(end_s * 1e9))
            z[f"{pre}c{c}_cross_events"] = np.int64(summ.total_cross_partition_events)
            z[f"{pre}c{c}_windows"] = np.int64(summ.total_windows)
            for q, o in enumerate(outs):
                pc = f"{pre}c{c}_p{q}_"
                for k in ("summaries", "entity_stats", "records", "sink_samples", "service_samples"):
                    z[pc + k] = o[k]
                if "sketches" in o:
                    z[pc + "sketch_state"] = o["sketches"]
            print(f"{name} cell {c}: {summ.total_windows} windows, {summ.total_cross_partition_events} cross-partition "
                  f"events, {[int(o['summaries']['events_processed'][0]) for o in outs]} events")
    np.savez_compressed(os.path.join(HERE, "lsweep_cells.npz"), **z)


if __name__ == "__main__":
    main()
