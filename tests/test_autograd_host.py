"""Host-side checks of the differentiable classifier's interface (no GPU needed): the C ABI version and entry points,
and the errors eot_logits raises before it would touch an engine."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_v9_declares_eot_entry_points():
    from dorpatch_b200 import _lib
    header = open(os.path.join(ROOT, "include", "dorpatch.h")).read()
    assert int(re.search(r"#define DP_ABI_VERSION (\d+)", header).group(1)) == 9 == _lib.ABI_VERSION
    for name in ("dp_eot_forward", "dp_eot_backward"):
        assert re.search(r"\b%s\(" % name, header) and name in _lib.SIGNATURES
    if os.path.exists(_lib.LIB_PATH):
        assert _lib.load().dp_abi_version() == 9


def _norm_model():
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    net = ResNetV2(num_classes=10, seed=0)
    return net, torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2")))


def test_eot_logits_on_cpu_raises_before_any_engine():
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    x = torch.rand(2, 3, 56, 56, requires_grad=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        eot_logits(model, x)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.module(x)                                    # NormModel's differentiable path
    with pytest.raises(RuntimeError, match="CUDA"):
        net((x - 0.5) / 0.5)                               # ResNetV2 on normalised input
    assert net._engines == {}


def test_eot_logits_rejects_foreign_modules():
    from dorpatch_b200.ops import eot_logits
    with pytest.raises(TypeError):
        eot_logits(torch.nn.Conv2d(3, 4, 1), torch.rand(1, 3, 56, 56))
