import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.lib()
    return oracle_lib


@pytest.fixture(scope="session")
def scene():
    """Small synthetic scene (833 nodes / 184 warps): octree + warp + edge blobs as numpy u8."""
    from synth_scene import SyntheticScene
    sc = SyntheticScene(n_cams=24, seed=0)
    nodes, trans, edges = sc.blobs()
    return dict(scene=sc, nodes=nodes, trans=trans, edges=edges, n_volumes=trans.size // 544)


def make_rays(scene, n_rays, seed=1234):
    o, d, cam = scene["scene"].rays(n_rays, seed)
    import torch
    dn = (torch.from_numpy(d) / torch.linalg.norm(torch.from_numpy(d), 2, -1, True)).numpy()
    return o, d, dn.astype(np.float32), cam


@pytest.fixture(scope="session")
def hash_params(scene):
    """Seeded table / primes / biases / MLP params shared by CPU and GPU tests (log2 table 15: small)."""
    rng = np.random.default_rng(7)
    log2 = 15
    V = scene["n_volumes"]
    pool = (1 << log2) * 16
    table = (rng.random((pool, 2), dtype=np.float32) * 2 - 1).astype(np.float16)
    prim = rng.integers(1 << 28, 1 << 30, size=(16, V, 3), dtype=np.int64).astype(np.int32) | 1
    bias = (rng.random((16 * V, 3), dtype=np.float32) * 1000 + 100).astype(np.float32)
    return dict(table=table, prim=prim, bias=bias, local_size=1 << log2, pool=pool, V=V)
