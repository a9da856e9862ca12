import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `pytest -m gpu`)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def c1(oracle):
    """C1 workload: cfg, synthetic weights (state_dict), pair, permutations, oracle result."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg

    cfg = workload_cfg("C1")
    model = init_synthetic_weights(bx.BufferX(cfg))
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    data = make_pair("C1", 0)
    perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], 0)
    res = oracle.register_pair(sd, cfg, data, perms, 0, keep=True)
    return dict(cfg=cfg, model=model, sd=sd, data=data, perms=perms, res=res)


@pytest.fixture(scope="session")
def c2_runs(oracle):
    """Lazy cache of full-size C2 oracle runs with the fitted CostNet (the configuration oracle/ref_check.py pins against
    the reference's own forward): ``c2_runs(seed, z_axes=None)`` -> dict(cfg, sd, data, perms, res)."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg

    cfg = workload_cfg("C2")
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    cache = {}

    def get(seed, z_axes=None, tag="free"):
        key = (seed, tag)
        if key not in cache:
            data = make_pair("C2", seed)
            perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], seed)
            res = oracle.register_pair(sd, cfg, data, perms, 0, keep=False, z_axes=z_axes)
            cache[key] = dict(cfg=cfg, sd=sd, model=model, data=data, perms=perms, res=res)
        return cache[key]

    return get
