import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "hades_golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def oracle():
    import hades_oracle
    return hades_oracle


@pytest.fixture(scope="session")
def coracle():
    import c_oracle
    c_oracle.lib()
    return c_oracle


@pytest.fixture(scope="session", params=["default", "throughput-kernel-only"])
def engine(request):
    """The CUDA engine.  No skip-on-failure: a GPU test without the native library or without an
    H100 must fail loudly.  Every test runs twice: with the default dispatch (digest batches up to 24 items per SM,
    3168 on an H100, take the lane-split small-batch kernel) and with that kernel disabled, so that both digest
    kernels see every shape."""
    import poseidon252_b200 as pb
    eng = pb.Engine(0)
    if request.param != "default":
        eng.set_small_batch_max(0)
    yield eng
    eng.close()


def mont(values):
    from poseidon252_b200.scalar import to_mont
    return to_mont(values)


def unmont(limbs):
    from poseidon252_b200.scalar import from_mont
    return from_mont(limbs)


def hx(s):
    return int(s, 16)


def edge_and_random_scalars(rng, n):
    """n scalars as Montgomery limbs: edge values (0, 1, p-1, R-related, KAT inputs) then random."""
    import hades_oracle as o
    from poseidon252_b200.scalar import random_scalars, to_mont
    edges = [0, 1, 2, o.P - 1, o.P - 2, o.R % o.P, (o.P - o.R) % o.P, (1 << 255) % o.P, (1 << 254), 5, 17] + o.kat_inputs()
    e = to_mont(edges[:n])
    if n > len(edges):
        return np.concatenate([e, random_scalars(rng, n - len(edges))], axis=0)
    return e
