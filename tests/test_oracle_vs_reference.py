"""Pin the oracle against a stored run of the UNMODIFIED reference (G8 in tests/golden/make_golden.py, which
runs the reference under the CPU shim of oracle/ref_shim.py): a 25-step targeted generate with dropout 2."""
import importlib.util
import os
import random

import numpy as np
import torch

from oracle import attack as OA

HERE = os.path.dirname(os.path.abspath(__file__))


def _mod():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "golden", "make_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_generate_live_bit_exact():
    mg = _mod()
    G = mg.load()
    tiny = mg.TinyNet().eval()
    xs = torch.rand(1, 3, 56, 56, generator=torch.Generator().manual_seed(21))
    kw = dict(patch_budget=0.12, n_classes=1000, targeted=True, y=torch.tensor([7]), max_iterations=25, sampling_size=3,
              dropout=2)
    random.seed(1234); torch.manual_seed(1234); np.random.seed(1234)
    log = []
    m, p = OA.generate(tiny, xs, log=log.append, **kw)
    assert np.array_equal(m.numpy(), G["g8_mask"]) and np.array_equal(p.numpy(), G["g8_pattern"])
    assert log == [str(s) for s in G["g8_log"]]
    assert np.array_equal(np.random.get_state()[1][:4], G["g8_rng_np"])
