import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree C-ABI library; built on demand (nvcc cross-compiles without a GPU)."""
    from mapdn_b200 import build
    return build.build()


def random_tree_net(n_bus, n_sgen, seed, with_taps=True):
    """Small random radial net exercising taps, line charging, bus shunts, scaling, parallel lines
    and a non-zero slack bus index."""
    from mapdn_b200.network import NetDesc
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n_bus)
    f, t = [], []
    for k in range(1, n_bus):
        f.append(perm[rng.integers(0, k)])
        t.append(perm[k])
    f, t = np.array(f), np.array(t)
    flip = rng.random(n_bus - 1) < 0.5
    f, t = np.where(flip, t, f), np.where(flip, f, t)
    r = rng.uniform(1e-3, 2e-2, n_bus - 1)
    x = r * rng.uniform(0.3, 2.0, n_bus - 1)
    b = rng.uniform(0, 2e-3, n_bus - 1)
    g = rng.uniform(0, 1e-4, n_bus - 1)
    tap = np.ones(n_bus - 1)
    is_line = np.ones(n_bus - 1, np.uint8)
    if with_taps:
        k = rng.choice(n_bus - 1, max(1, (n_bus - 1) // 6), replace=False)
        tap[k] = rng.uniform(0.95, 1.05, len(k))
        is_line[k] = 0
    # one parallel twin and one out-of-service branch
    f = np.r_[f, f[0], f[1]]; t = np.r_[t, t[0], t[1]]
    r = np.r_[r, r[0] * 1.3, r[1]]; x = np.r_[x, x[0] * 0.9, x[1]]
    b = np.r_[b, 0.0, 0.0]; g = np.r_[g, 0.0, 0.0]; tap = np.r_[tap, tap[0], 1.0]
    is_line = np.r_[is_line, is_line[0], 1].astype(np.uint8)
    status = np.ones(n_bus + 1, np.uint8); status[-1] = 0
    n_zone = 3
    zone = rng.integers(0, n_zone + 1, n_bus).astype(np.int32)
    sgen_bus = rng.choice(n_bus, n_sgen, replace=False).astype(np.int32)
    zone[sgen_bus] = np.maximum(zone[sgen_bus], 1)
    n_load = n_bus + 3
    load_bus = np.r_[np.arange(n_bus), rng.integers(0, n_bus, 3)].astype(np.int32)
    return NetDesc(base_mva=10.0, n_bus=n_bus, slack_bus=int(perm[0]), slack_vm=1.02, slack_va_deg=3.0,
                   br_from=f, br_to=t, br_r=r, br_x=x, br_b=b, br_g=g, br_tap=tap, br_status=status,
                   br_is_line=is_line, bus_gs=rng.uniform(0, 0.05, n_bus), bus_bs=rng.uniform(-0.05, 0.05, n_bus),
                   load_bus=load_bus, load_scaling=rng.uniform(0.8, 1.2, n_load),
                   sgen_bus=sgen_bus, sgen_zone=zone[sgen_bus], sgen_scaling=rng.uniform(0.9, 1.1, n_sgen),
                   bus_zone=zone, name=f"rand{n_bus}")
