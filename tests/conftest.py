import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    try:
        import torch
        torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    except Exception:
        pass


@pytest.fixture(scope="session")
def oracle_params():
    from oracle import resnetv2 as R
    return R.random_init(seed=0, affine_jitter=0.1)


@pytest.fixture(scope="session")
def oracle_net(oracle_params):
    import torch
    from oracle import resnetv2 as R
    # torch-CPU convolutions get much slower when oversubscribed (128 threads on the GPU box)
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    return R.OracleNet(oracle_params, weights_require_grad=False).eval()


_ENGINES = {}


@pytest.fixture(scope="session")
def engine_factory(oracle_params):
    """Engines are expensive (workspace + cuDNN autotune); cache per configuration."""
    from dorpatch_b200.engine import Engine

    def make(img=112, precision="fp32", chunk=8, max_images=4):
        key = (img, precision, chunk, max_images)
        if key not in _ENGINES:
            e = Engine(img=img, precision=precision, chunk=chunk, max_images=max_images, autotune=False)
            e.load_state_dict(oracle_params)
            _ENGINES[key] = e
        return _ENGINES[key]

    yield make
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()
