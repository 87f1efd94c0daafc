"""The C-ABI library loads and exports every symbol include/hs_b200.h declares (no GPU needed)."""
import ctypes as C
import os
import re

import pytest

import happysim_b200 as hs
from happysim_b200 import engine, _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    return engine.load_library()


def declared_functions():
    src = open(os.path.join(ROOT, "include", "hs_b200.h")).read()
    body = src[src.index("/* ---- entry points"):]
    return sorted(set(re.findall(r"^(?:int|uint32_t|void)\s+(hs_\w+)\s*\(", body, flags=re.M)))


def test_every_declared_entry_point_is_exported(lib):
    names = declared_functions()
    assert len(names) >= 13
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/hs_b200.h but not exported"
    assert sorted(engine.EXPORTED_SYMBOLS) == names


def test_version_and_struct_layouts(lib):
    assert lib.hs_version() == A.HS_ABI_VERSION
    src = open(os.path.join(ROOT, "include", "hs_b200.h")).read()
    assert "hs_entity_desc;      /* 48 bytes */" in src and C.sizeof(A.EntityDesc) == 48
    assert C.sizeof(A.ReplicaSummary) == 56 and C.sizeof(A.EntityStats) == 64
    assert C.sizeof(A.EventRecord) == 16 and C.sizeof(A.SinkSample) == 16
    assert C.sizeof(A.LinkDesc) == 24 and A.XEVENT_DTYPE.itemsize == 40          # hs_link_desc, hs_xevent
    assert C.sizeof(A.Totals) == 8 * (A.HS_TOTALS_I64 + A.HS_TOTALS_F64_SUM + 2)
    assert f"#define HS_ABI_VERSION {A.HS_ABI_VERSION}u" in src
    assert "hs_launch_info;      /* 32 bytes */" in src and C.sizeof(A.LaunchInfo) == 32


def test_a_library_of_another_abi_version_fails_the_version_check(tmp_path):
    """A library built from older sources exports an older hs_version and lacks newer entry points: loading it names
    the version mismatch, not the first missing symbol."""
    import shutil
    import subprocess
    cc = shutil.which(os.environ.get("CC", "cc")) or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "stale.c"
    src.write_text(f"unsigned int hs_version(void) {{ return {A.HS_ABI_VERSION - 1}u; }}\n")
    so = tmp_path / "libstale.so"
    subprocess.check_call([cc, "-shared", "-fPIC", "-o", str(so), str(src)])
    with pytest.raises(engine.EngineError, match=f"ABI version {A.HS_ABI_VERSION - 1}, this package needs {A.HS_ABI_VERSION}"):
        engine.load_library(str(so))


def test_engine_fails_loudly_without_a_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine(0)
    assert ei.value.code == A.HS_ERR_NO_DEVICE


def test_model_validation_errors(lib):
    engine.validate_model(hs.mm1())
    engine.validate_model(hs.lb_round_robin(4, 32.0))
    bad = hs.mm1(); bad.entities["d0"][0] = 0.0                     # zero rate (arrival_time_provider.py:75)
    with pytest.raises(engine.EngineError, match="rate must be > 0"):
        engine.validate_model(bad)
    bad = hs.mm1(); bad.entities["i0"][1] = 0                       # FixedConcurrency(0) (concurrency.py:86)
    with pytest.raises(engine.EngineError, match="max_concurrent must be >= 1"):
        engine.validate_model(bad)
    bad = hs.mm1(); bad.entities["target"][0] = 9
    with pytest.raises(engine.EngineError, match="out of range"):
        engine.validate_model(bad)
    bad = hs.lb_round_robin(4, 32.0); bad.backends[2] = 0           # a Source as backend
    with pytest.raises(engine.EngineError, match="must be a Server, CachingServer, Sink or Counter"):
        engine.validate_model(bad)
