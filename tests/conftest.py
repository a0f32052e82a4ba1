"""pytest configuration: markers + shared fixtures.

`-m "not gpu"`  : oracle vs golden vectors, host logic, C-ABI symbol checks, gloo sharding tests (CPU).
`-m gpu`        : parity of the CUDA path (through the C-ABI) against the oracle and the goldens.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a host without a CUDA device (or without the built library) skips the gpu-marked tests
    instead of failing in the first one; `-m gpu` on a GPU machine runs them (there is no CPU fallback to fall into)."""
    reason = None
    try:
        import torch

        if not torch.cuda.is_available():
            reason = "no CUDA device"
    except Exception as e:  # pragma: no cover
        reason = f"torch unavailable: {e}"
    if reason is None and not os.path.isfile(os.path.join(ROOT, "moleculekit_b200", "lib", "libmkb200.so")):
        reason = "moleculekit_b200/lib/libmkb200.so not built"
    if reason:
        skip = pytest.mark.skip(reason=reason)
        for item in items:
            if "gpu" in item.keywords:
                item.add_marker(skip)


def _npz(name):
    with np.load(os.path.join(GOLDEN, name), allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def g_voxel3ptb():
    return _npz("voxel_3ptb.npz")


@pytest.fixture(scope="session")
def g_voxelsmall():
    return _npz("voxel_small.npz")


@pytest.fixture(scope="session")
def g_traj():
    return _npz("traj20.npz")


@pytest.fixture(scope="session")
def g_3ptb():
    return _npz("pdb_3ptb.npz")


@pytest.fixture(scope="session")
def g_5vl5():
    return _npz("pdb_5vl5.npz")


@pytest.fixture(scope="session")
def g_raw():
    return _npz("rawkernels.npz")


@pytest.fixture(scope="session")
def g_bonds():
    return _npz("bonds.npz")


@pytest.fixture(scope="session")
def g_xtc():
    g = _npz("xtc.npz")
    g["_dir"] = os.path.join(GOLDEN, "xtc")
    return g


@pytest.fixture(scope="session")
def g_interactions():
    return _npz("interactions.npz")


@pytest.fixture(scope="session")
def g_within():
    return _npz("within.npz")


@pytest.fixture(scope="session")
def g_rotate():
    return _npz("rotate.npz")


@pytest.fixture(scope="session")
def g_wrap():
    return _npz("wrap.npz")


@pytest.fixture(scope="session")
def g_tric():
    return _npz("tric.npz")


@pytest.fixture(scope="session")
def g_rings():
    return _npz("rings.npz")


@pytest.fixture(scope="session")
def g_waterbridge():
    return _npz("waterbridge.npz")


@pytest.fixture(scope="session")
def g_hbonds():
    return _npz("hbonds.npz")


@pytest.fixture(scope="session")
def oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


@pytest.fixture(scope="session")
def refmods():
    """The reference's own compiled kernels (oracle/_ref) when available, else None."""
    from oracle import build_ref

    try:
        build_ref.build(verbose=False)
    except Exception:
        pass
    return build_ref.load()
