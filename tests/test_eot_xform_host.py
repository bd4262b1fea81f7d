"""Host-side checks of affine / colour EOT in the differentiable classifier (no GPU needed): the C ABI entry point, and
the errors eot_logits(..., xforms=...) raises before it would touch an engine."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_and_signatures_declare_eot_forward_xform():
    from dorpatch_b200 import _lib
    header = open(os.path.join(ROOT, "include", "dorpatch.h")).read()
    assert int(re.search(r"#define DP_ABI_VERSION (\d+)", header).group(1)) == 9 == _lib.ABI_VERSION
    m = re.search(r"int32_t dp_eot_forward_xform\(([^)]*)\)", header)
    assert m, "dp_eot_forward_xform is not declared"
    assert len(m.group(1).split(",")) == 8
    assert "dp_eot_forward_xform" in _lib.SIGNATURES
    restype, argtypes = _lib.SIGNATURES["dp_eot_forward_xform"]
    assert len(argtypes) == 8
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        assert lib.dp_abi_version() == 9
        assert hasattr(lib, "dp_eot_forward_xform")


def _norm_model():
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    net = ResNetV2(num_classes=10, seed=0)
    return net, torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2")))


def _xforms(B, S, seed=0):
    from dorpatch_b200 import eot
    return eot.sample(np.random.RandomState(seed), B, S, 0.1, 0.1)


def test_eot_logits_xforms_on_cpu_raises_before_any_engine():
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    x = torch.rand(2, 3, 56, 56, requires_grad=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        eot_logits(model, x, None, 4, xforms=_xforms(2, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        eot_logits(model, x, None, 4, xforms=torch.from_numpy(_xforms(2, 4)))
    assert net._engines == {}


def test_eot_logits_xforms_rejects_foreign_modules():
    from dorpatch_b200.ops import eot_logits
    with pytest.raises(TypeError):
        eot_logits(torch.nn.Conv2d(3, 4, 1), torch.rand(1, 3, 56, 56), None, 2, xforms=_xforms(1, 2))


@pytest.mark.parametrize("bad", [
    np.zeros((2, 4, 7), np.float32),          # 7 numbers per sample
    np.zeros((2, 3, 8), np.float32),          # S does not match
    np.zeros((3, 4, 8), np.float32),          # B does not match
    np.zeros((8, 8), np.float32),             # flattened
    np.zeros((2, 4, 8, 1), np.float32),       # extra axis
])
def test_eot_logits_xforms_wrong_shape_raises_before_any_engine(bad):
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    x = torch.rand(2, 3, 56, 56, requires_grad=True)
    with pytest.raises(ValueError, match="xforms"):
        eot_logits(model, x, None, 4, xforms=bad)
    with pytest.raises(ValueError, match="xforms"):
        eot_logits(model, x, None, 4, xforms=torch.from_numpy(bad))
    assert net._engines == {}


@pytest.mark.parametrize("bad", [
    np.zeros((2, 4, 8), np.int32),
    np.zeros((2, 4, 8), np.bool_),
    torch.zeros((2, 4, 8), dtype=torch.int64),
    torch.zeros((2, 4, 8), dtype=torch.complex64),
])
def test_eot_logits_xforms_wrong_dtype_raises_before_any_engine(bad):
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    x = torch.rand(2, 3, 56, 56, requires_grad=True)
    with pytest.raises(TypeError, match="xforms"):
        eot_logits(model, x, None, 4, xforms=bad)
    assert net._engines == {}
