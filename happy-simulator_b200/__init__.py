"""happysim_b200 -- H100-native engine behind the happy-simulator modelling API.

The hot path of the reference (``Simulation.run()``'s pop-invoke-push loop over
a heapq of Python ``Event`` objects, happysimulator/core/simulation.py:449-505)
runs here as hand-written sm_90a CUDA behind a C-ABI (include/hs_b200.h);
this package is the thin Python host side: the modelling classes users already
write against, the lowering of their object graph to a flat model table, and
the ctypes binding.  There is NO CPU fallback: without the CUDA library and a
GPU, ``run()`` raises.
"""
from . import _abi  # noqa: F401
from . import engine  # noqa: F401
from .model import FlatModel, ModelBuilder, mm1, lb_round_robin, lb_key_table, mmc_sweep  # noqa: F401

__version__ = "0.1.0"

from .lowering import lower, consistent_hash_table, hll_table, cms_table, bloom_table, zipf_cdf, UnsupportedModelError  # noqa: F401,E402
from .sketching import (HyperLogLog, CountMinSketch, BloomFilter, TopK, ReservoirSampler, SketchCollector, TopKCollector,  # noqa: F401,E402
                        KeyExtractor, FrequencyEstimate, TDigest, QuantileEstimator, LatencyExtractor)  # noqa: F401,E402
from .api import (  # noqa: F401,E402
    Instant, Duration, Entity, Source, SimpleEventProvider, ConstantRateProfile, ConstantArrivalTimeProvider,
    PoissonArrivalTimeProvider, ConstantLatency, ExponentialLatency, FIFOQueue, LIFOQueue, FixedConcurrency,
    Server, ServerStats, CachingServer, CachingServerStats, Sink, Counter, LoadBalancer, LoadBalancerStats, RoundRobin, ConsistentHash,
    UniformKeyContext, ZipfKeyContext, StepProfile, Simulation, SimulationSummary, EntitySummary, QueueStats, ParallelRunner, RunConfig,
    ParallelResult, seed, run_lowered, LinearRampProfile, SpikeProfile,
)
from . import api  # noqa: F401,E402
from .instrumentation import Data, BucketedData, LatencyTracker, ThroughputTracker, Probe  # noqa: F401,E402
from .parallel import SimulationPartition, PartitionLink, ParallelSimulation, ParallelSimulationSummary  # noqa: F401,E402
from .hook import install, uninstall, stats as install_stats  # noqa: F401,E402
