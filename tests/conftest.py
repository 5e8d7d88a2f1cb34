import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

GOLDEN = ROOT / "tests" / "golden"

# (file stem, oracle arithmetic family that produced it: 1 = FMA build, 0 = SSE / *_Gen_SSE)
GOLDEN_FILES = [
    ("primates_gtr_g4_fma", 1),
    ("primates_gtr_g4_sse", 0),
    ("primates_gtr_ig4_fma", 1),
    ("primates_gtr_eq_fma", 1),
    ("ovomucoids_wag_g4_sse", 0),
    ("replicase_m0_sse", 0),
    ("primates_hky_g4_fma", 1),      # nst=2: closed-form model, eigensystem sent inline
    ("primates_f81_i_fma", 1),       # nst=1 + pInvar
    ("replicase_ny98_sse", 0),       # codon NY98: one eigensystem per omega category (TiProbs_GenCov, *_NY98)
    ("cynmix_part_fma", 1),          # cynmix, 4 unlinked GTR+I+G4 DNA partitions (32 taxa), interleaved evaluations
    ("cynmix_full_fma", 1),          # cynmix, all 5 partitions: morphology Mk+G4 (variable-state *_Std family) + the 4 DNA ones
]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def oracle_lib():
    from mrbayes_b200 import abi
    if not abi.ORACLE_LIB.exists():
        import subprocess
        subprocess.run(["make", "-C", str(ROOT / "oracle"), "oracle"], check=True)
    return abi.oracle_library()


@pytest.fixture(scope="session")
def engine_lib():
    """The CUDA engine.  GPU tests must run the native path: a missing .so or a missing
    device is an error, never a skip to a fallback."""
    from mrbayes_b200 import abi
    lib = abi.engine_library()
    assert lib.fn("device_count")() >= 1, "no sm_90 device: the engine has no CPU fallback"
    return lib
