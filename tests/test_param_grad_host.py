"""Host-side checks of weight gradients through the native classifier (no GPU needed): the two C ABI entry points
(dp_eot_backward_params, dp_engine_load_weights_dev) and the errors eot_logits(..., param_grads=True) raises before it
would touch an engine."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,nargs", [("dp_eot_backward_params", 8), ("dp_engine_load_weights_dev", 6),
                                        ("dp_debug_stem_wgrad", 6), ("dp_debug_gn_wgrad", 12),
                                        ("dp_debug_ws_backward", 10)])
def test_header_and_signatures_declare_param_grad_entries(name, nargs):
    from dorpatch_b200 import _lib
    header = open(os.path.join(ROOT, "include", "dorpatch.h")).read()
    assert int(re.search(r"#define DP_ABI_VERSION (\d+)", header).group(1)) == 9 == _lib.ABI_VERSION
    m = re.search(r"int32_t %s\(([^)]*)\)" % name, header)
    assert m, "%s is not declared" % name
    assert len(m.group(1).split(",")) == nargs
    restype, argtypes = _lib.SIGNATURES[name]
    assert len(argtypes) == nargs
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        assert lib.dp_abi_version() == 9
        assert hasattr(lib, name)


def _norm_model():
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    net = ResNetV2(num_classes=10, seed=0)
    return net, torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2")))


def test_param_grads_on_cpu_raises_before_any_engine():
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    with pytest.raises(RuntimeError, match="CUDA"):
        eot_logits(model, torch.rand(2, 3, 56, 56), None, 1, param_grads=True)
    net.param_grads_(True)
    with pytest.raises(RuntimeError, match="CUDA"):
        net(torch.rand(2, 3, 56, 56))
    assert net._engines == {}


@pytest.mark.parametrize("bad", [1, "yes", None, torch.tensor(True)])
def test_param_grads_must_be_a_bool(bad):
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    with pytest.raises(TypeError, match="param_grads"):
        eot_logits(model, torch.rand(1, 3, 56, 56), None, 1, param_grads=bad)
    assert net._engines == {}


def test_param_grads_needs_fp32_parameters():
    from dorpatch_b200.ops import eot_logits
    net, model = _norm_model()
    net.norm.weight.data = net.norm.weight.data.double()
    with pytest.raises(TypeError, match="norm.weight"):
        eot_logits(model, torch.rand(1, 3, 56, 56), None, 1, param_grads=True)
    assert net._engines == {}


def test_param_grads_rejects_foreign_modules():
    from dorpatch_b200.ops import eot_logits
    with pytest.raises(TypeError):
        eot_logits(torch.nn.Conv2d(3, 4, 1), torch.rand(1, 3, 56, 56), None, 1, param_grads=True)


def test_param_grads_mode_is_off_by_default_and_chains():
    net, _ = _norm_model()
    assert net._param_grads is False
    assert net.param_grads_(True) is net and net._param_grads is True
    assert net.param_grads_(False)._param_grads is False
