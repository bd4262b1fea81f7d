"""dp_engine_launch_count against the kernels the GPU actually ran, as CUPTI records them through torch.profiler
(activity tracing).  Every kernel of this library is defined inside `namespace dp`, so its demangled name contains
"dp::"; the counter must equal the number of those kernels, plus one per cuDNN / cublasLt call.

Op-level hooks make no library call: there the counter delta equals the dp:: kernels exactly.  Whole-network calls run on
an fp32 engine at 112 px with the engine profiler on (one lane), where the library calls are exactly the regions of
the library categories below, so delta = dp:: kernels + those regions."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# Profiler categories of the engine's cuDNN / cublasLt calls (conv_fwd, conv_bwd, conv_wgrad, gemm, wgrad_gemm in
# engine.cu).  At fp32 the stem is cuDNN, so its categories are library calls too.  fc_wgrad also holds the bias
# gradient's column-sum kernel (one region per chunk when head.fc.bias is wanted).
LIBRARY = {"stem_conv_fwd", "stem_conv_bwd", "stem_wgrad", "conv3x3_fwd", "conv3x3_bwd", "conv3x3_wgrad",
           "gemm1x1_fwd", "gemm1x1_bwd", "gemm1x1_wgrad", "fc_fwd", "fc_bwd", "fc_wgrad"}
# Categories whose regions hold only kernels of this library (CUPTI counts those).  A category in neither set fails
# the test, so a new one has to be classified here.
OWN = {"expand_k1", "expand_affine", "reduce_k1t", "reduce_affine", "paste", "struct", "maskreg", "cw_k4", "update_k3",
       "maxpool_fwd", "maxpool_bwd", "stem_bwd_reduce", "gn_relu_fwd", "gn_relu_bwd", "gn_stats", "gn_gemm1x1_fwd",
       "subsample", "head_fwd", "head_bwd", "gn_affine_wgrad", "gn_apply_wgrad", "ws_wgrad", "vec_wgrad"}


OWN_KERNEL = re.compile(r"(?<![A-Za-z0-9_])dp::")


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _rand(shape, seed, dtype=torch.float32):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 2 - 1).to(dtype).to(DEV)


def _counted(e, fn):
    """(launch-count delta of fn(), dp:: kernels CUPTI recorded during fn()).  A torch kernel runs first inside the
    trace: when the trace holds no CUDA kernel at all, CUPTI is not recording here and the test skips."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(4096, device=DEV).mul_(3.0)
        torch.cuda.synchronize()
        l0 = e.launch_count
        fn()
        torch.cuda.synchronize()
        delta = e.launch_count - l0
    kernels = [ev.name for ev in prof.events() if ev.device_type == DeviceType.CUDA]
    if not any(not OWN_KERNEL.search(k) and "memcpy" not in k.lower() and "memset" not in k.lower() for k in kernels):
        pytest.skip("torch.profiler recorded no CUDA kernel for a torch op: no CUPTI activity records on this machine")
    return delta, sum(bool(OWN_KERNEL.search(k)) for k in kernels)


def _engine(oracle_params, **kw):
    from dorpatch_b200.engine import Engine
    e = Engine(device=0, autotune=False, **kw)
    e.load_state_dict(oracle_params)
    return e


@pytest.fixture(scope="module")
def bf16_engine(oracle_params):
    e = _engine(oracle_params, img=224, precision="bf16", chunk=8, max_images=2)
    yield e
    e.close()


@pytest.fixture(scope="module")
def fp32_engine(oracle_params):
    saved = os.environ.get("DORPATCH_GRAPH")
    os.environ["DORPATCH_GRAPH"] = "0"   # dp_attack_grad eagerly: its launches are the ones traced
    try:
        e = _engine(oracle_params, img=112, precision="fp32", chunk=4, max_images=2)
    finally:
        if saved is None:
            os.environ.pop("DORPATCH_GRAPH")
        else:
            os.environ["DORPATCH_GRAPH"] = saved
    yield e
    e.close()


# (3136, 64) takes the one-kernel cluster plan, (7056, 256) the two-pass fallback (tests/test_gpu_ops.py)
@pytest.mark.parametrize("P,Cc,fwd_kernels", [(3136, 64, 1), (7056, 256, 2)])
@pytest.mark.parametrize("mode", ["stats", "fwd", "fwd_bwd"])
def test_groupnorm_hook(bf16_engine, P, Cc, fwd_kernels, mode):
    from dorpatch_b200 import _lib
    e, N = bf16_engine, 3
    x, dy = _rand((N, P, Cc), 1, torch.bfloat16), _rand((N, P, Cc), 2, torch.bfloat16)
    gamma, beta = 1.0 + 0.3 * _rand((Cc,), 3), 0.3 * _rand((Cc,), 4)
    y, dx, stats = torch.empty_like(x), torch.empty_like(x), torch.empty(N, 32, 2, device=DEV)
    y_, dy_, dx_ = (None, None, None) if mode == "stats" else (y, dy if mode == "fwd_bwd" else None, dx)

    def call():
        _lib.check(e.lib.dp_debug_gn(e.handle, _ptr(x), _ptr(dy_), None, _ptr(gamma), _ptr(beta), 1, _ptr(y_), _ptr(dx_),
                                     _ptr(stats), N, P, Cc, e._stream()))
    delta, dp_kernels = _counted(e, call)
    if mode == "fwd":   # the shape takes the GroupNorm path this case is meant to cover
        assert dp_kernels == fwd_kernels
    assert delta == dp_kernels > 0


def test_patch_helpers(bf16_engine):
    from dorpatch_b200 import masks as PM
    e, B, S, H = bf16_engine, 2, 3, 224
    x, p, m = _rand((B, 3, H, H), 5).abs(), _rand((B, 3, H, H), 6).abs(), _rand((B, 1, H, H), 7).abs()
    rects = PM.gather(PM.universe(H, 2), np.array([[1, 40, 900], [7, 300, 2000]]))
    for fn in (lambda: e.paste(x, m, p, 4.0, out=torch.empty_like(x)), lambda: e.window_sum(m, 7, square=True),
               lambda: e.expand(x, S, rects)):
        delta, dp_kernels = _counted(e, fn)
        assert delta == dp_kernels > 0


def test_failed_set_update(bf16_engine):
    e, B, S = bf16_engine, 2, 5
    e.failed_reset(100)
    idx = np.arange(B * S, dtype=np.int32).reshape(B, S) * 3
    loss = np.linspace(-1, 1, B * S).astype(np.float32).reshape(B, S)
    delta, dp_kernels = _counted(e, lambda: e.failed_update(idx, np.full(B, S, np.int32), np.ones(B, np.uint8), loss=loss))
    assert delta == dp_kernels > 0


@pytest.mark.parametrize("backward", [False, True])
def test_maxpool_hook(bf16_engine, backward):
    from dorpatch_b200 import _lib
    e, N, Hs, Cc = bf16_engine, 2, 112, 64
    x = _rand((N, Hs, Hs, Cc), 8, torch.bfloat16)
    y = torch.empty(N, Hs // 2, Hs // 2, Cc, dtype=torch.bfloat16, device=DEV)
    amax = torch.empty(N, Hs // 2, Hs // 2, Cc, dtype=torch.int8, device=DEV)
    dy = _rand(y.shape, 9, torch.bfloat16) if backward else None
    dx = torch.empty_like(x) if backward else None
    delta, dp_kernels = _counted(e, lambda: _lib.check(e.lib.dp_debug_maxpool(
        e.handle, _ptr(x), _ptr(y), _ptr(amax), _ptr(dy), _ptr(dx), N, Hs, Cc, e._stream())))
    assert delta == dp_kernels > 0


def test_stem_wgrad_hook(bf16_engine):
    from dorpatch_b200 import _lib
    e, N, H = bf16_engine, 2, 224
    x, dy = _rand((N, H, H, 3), 10, torch.bfloat16), _rand((N, H // 2, H // 2, 64), 11, torch.bfloat16)
    dw = torch.empty(64, 7, 7, 3, device=DEV)
    delta, dp_kernels = _counted(e, lambda: _lib.check(e.lib.dp_debug_stem_wgrad(
        e.handle, _ptr(x), _ptr(dy), N, _ptr(dw), e._stream())))
    assert delta == dp_kernels > 0


@pytest.mark.parametrize("apply", [False, True])
def test_gn_wgrad_hook(bf16_engine, apply):
    from dorpatch_b200 import _lib
    e, N, P, Cc = bf16_engine, 2, 784, 128
    x, dy = _rand((N, P, Cc), 12, torch.bfloat16), _rand((N, P, Cc), 13, torch.bfloat16)
    gamma, beta = 1.0 + 0.3 * _rand((Cc,), 14), 0.3 * _rand((Cc,), 15)
    stats = torch.stack([torch.zeros(N, 32), torch.ones(N, 32)], -1).contiguous().to(DEV)
    dgb = torch.empty(2 * Cc, device=DEV)
    y = torch.empty_like(x) if apply else None
    delta, dp_kernels = _counted(e, lambda: _lib.check(e.lib.dp_debug_gn_wgrad(
        e.handle, _ptr(x), _ptr(dy), _ptr(gamma), _ptr(beta), _ptr(stats), N, P, Cc, _ptr(dgb), _ptr(y), e._stream())))
    assert delta == dp_kernels > 0


@pytest.mark.parametrize("name", ["stages.0.blocks.1.conv1.weight", "stem.conv.weight"])
def test_weight_reload(bf16_engine, oracle_params, name):
    e = bf16_engine
    w = torch.as_tensor(oracle_params[name]).float().to(DEV)
    delta, dp_kernels = _counted(e, lambda: e.load_state_dict_dev({name: w}))
    assert delta == dp_kernels > 0


def test_whole_network_calls(fp32_engine):
    from dorpatch_b200 import masks as PM
    from dorpatch_b200.resnetv2 import param_shapes
    e, B, S, H, K = fp32_engine, 2, 4, 112, 1000
    N, chunks = B * S, (B * S + 3) // 4
    g = torch.Generator().manual_seed(20)
    img, x, p = (torch.rand(B, 3, H, H, generator=g).to(DEV) for _ in range(3))
    m = torch.rand(B, 1, H, H, generator=g).to(DEV)
    dlog = torch.randn(N, K, generator=g).to(DEV)
    rects = PM.gather(PM.universe(H, 2), np.random.RandomState(21).randint(0, 2520, (B, S)))
    G = torch.zeros(B, 3, H, H, device=DEV)
    shapes = param_shapes(K)
    grads = [torch.zeros(shapes[n], device=DEV) for n in shapes]
    lr, structured, coeff = np.full(B, 0.01, np.float32), np.full(B, 1e-3, np.float32), np.full(B, 1e-5, np.float32)
    calls = [
        ("predict", lambda: e.predict(img, S, rects), 0),
        ("attack_grad", lambda: e.attack_grad(x, m, p, rects, np.array([3, 9]), [True, False], 0.1, 4.0, 0, G), 0),
        ("attack_update", lambda: e.attack_update(x, m, p, G, lr, structured, coeff, 1e-3, 0), 0),
        ("eot_forward", lambda: e.eot_forward(img, S, rects), 0),
        ("eot_backward", lambda: e.eot_backward(dlog), 0),
        ("eot_backward_params", lambda: e.eot_backward_params(dlog, list(shapes), grads, grad_img=True), chunks),
    ]
    for name, fn, fc_bias_sums in calls:
        e.profile(True, reset=True)
        try:
            delta, dp_kernels = _counted(e, fn)
            prof = e.profile_read()
        finally:
            e.profile(False)
        unknown = set(prof) - LIBRARY - OWN
        assert not unknown, (name, unknown)
        library = sum(d["count"] for c, d in prof.items() if c in LIBRARY) - fc_bias_sums
        print(name, "launches", delta, "dp:: kernels", dp_kernels, "library calls", library)
        assert dp_kernels > 0
        assert delta == dp_kernels + library, (name, delta, dp_kernels, library)
