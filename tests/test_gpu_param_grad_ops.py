"""Operator-level checks of the weight-gradient pass's hand-written kernels against fp64 torch restatements on the same
rounded operands (dp_debug_gn_wgrad, dp_debug_ws_backward; the bf16 stem kernel is in test_gpu_param_grad.py)."""
import ctypes as C

import pytest
import torch

from dorpatch_b200 import _lib
from oracle import resnetv2 as OR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-300))


@pytest.fixture(scope="module")
def engines():
    from dorpatch_b200.engine import Engine
    made = {}

    def get(precision):
        if precision not in made:
            e = Engine(img=56, precision=precision, chunk=4, max_images=1, autotune=False)
            e.load_state_dict(OR.random_init(seed=0))
            made[precision] = e
        return made[precision]
    yield get
    for e in made.values():
        e.close()
    torch.cuda.empty_cache()


# every (pixels, channels) class the engine's GroupNorms run at 224 px (norm1 / norm2 / norm3 of each stage, the head)
SHAPES = [(3136, 64), (3136, 256), (784, 128), (784, 256), (784, 512), (196, 256), (196, 512), (196, 1024),
          (49, 512), (49, 1024), (49, 2048)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("P,Cc", SHAPES)
def test_gn_wgrad_vs_fp64(engines, precision, P, Cc):
    """dgamma / dbeta (per-sample partials + fixed-order column sum) within 1e-5 relative L2 of fp64 on the same rounded
    x / dy and stats, the ReLU gate evaluated as the kernel does (sign of gamma*rstd*x + beta - mean*gamma*rstd on the
    fp32 constants; some gammas negative); relu(gn(x)) re-applied within one ulp of the activation dtype."""
    e = engines(precision)
    dt = torch.bfloat16 if precision == "bf16" else torch.float32
    N = 2
    g = torch.Generator().manual_seed(P * 7 + Cc)
    x = (torch.randn(N, P, Cc, generator=g) * 1.5 + 0.3).to(dt)
    dy = torch.randn(N, P, Cc, generator=g).to(dt)
    gamma = torch.randn(Cc, generator=g) * 0.5 + 0.8
    beta = torch.randn(Cc, generator=g) * 0.3
    xg = x.double().reshape(N, P, 32, Cc // 32)
    mean = xg.mean((1, 3)).float()
    rstd = (1.0 / torch.sqrt(xg.var((1, 3), unbiased=False) + 1e-5)).float()
    stats = torch.stack([mean, rstd], -1).contiguous()                                   # [N, 32, 2]
    dgb = torch.empty(2 * Cc, device=DEV)
    y = torch.empty(N, P, Cc, dtype=dt, device=DEV)
    xd, dyd, gd, bd, sd = x.to(DEV), dy.to(DEV), gamma.to(DEV), beta.to(DEV), stats.to(DEV)
    _lib.check(e.lib.dp_debug_gn_wgrad(e.handle, _ptr(xd), _ptr(dyd), _ptr(gd), _ptr(bd), _ptr(sd), N, P, Cc, _ptr(dgb),
                                       _ptr(y), e._stream()))
    torch.cuda.synchronize()
    grp = torch.arange(Cc) // (Cc // 32)
    mu, rs = mean[:, grp][:, None, :], rstd[:, grp][:, None, :]                          # [N, 1, C] fp32
    s1 = rs * gamma                                                                      # the kernel's fp32 constants
    got = dgb.cpu().double()
    best = None
    # beta - mean * s1: two roundings, or one when the compiler contracts it into an fma -- either is the kernel's
    for s0 in (beta - mu * s1, (beta.double() - mu.double() * s1.double()).float()):
        pre = s1.double() * x.double() + s0.double()                                     # exact sign of the fp32 fma
        dyg = torch.where(pre > 0, dy.double(), torch.zeros((), dtype=torch.float64))
        xhat = (x.double() - mu.double()) * rs.double()
        rg, rb = _rel(got[:Cc], (dyg * xhat).sum((0, 1))), _rel(got[Cc:], dyg.sum((0, 1)))
        ref_y = pre.clamp_min(0)
        tol = ref_y * (2 ** -8 if dt == torch.bfloat16 else 2 ** -23) + 1e-6
        err_y = ((y.cpu().double() - ref_y).abs() - tol).max().item()
        if best is None or max(rg, rb) < max(best[0], best[1]):
            best = (rg, rb, err_y)
    rg, rb, err_y = best
    print(precision, P, Cc, "dgamma", rg, "dbeta", rb, "y excess over one ulp", err_y)
    assert rg <= 1e-5 and rb <= 1e-5
    assert err_y <= 0


@pytest.mark.parametrize("O,I,k,Ipad,scale", [
    (64, 3, 7, 4, 0.05),       # fp32 / tf32 stem: cuDNN's channel-padded filter
    (64, 3, 7, 8, 0.05),       # bf16 engine's stem filter (own-stem accumulator layout)
    (64, 64, 3, 64, 0.05),
    (256, 64, 1, 64, 0.05),
    (512, 512, 3, 512, 0.02),
    (128, 256, 1, 256, 1e-4),  # variance 1e-8: the standardisation's eps is half of it
])
def test_ws_backward_vs_autograd(engines, O, I, k, Ipad, scale):
    """The weight-standardisation adjoint against fp64 autograd through oracle.resnetv2.standardize (eps 1e-8): within
    1e-5 relative L2; the pad channels of the KRSC gradient carry garbage that must not leak; two lane halves."""
    e = engines("fp32")
    g = torch.Generator().manual_seed(O + I + k + Ipad)
    w = torch.randn(O, I, k, k, generator=g) * scale + scale * 0.3
    gk = torch.randn(O, k, k, Ipad, generator=g)                                         # d/d(standardised w), KRSC
    ga = torch.randn(O, k, k, Ipad, generator=g)
    gb = gk - ga
    out = torch.empty(O, I, k, k, device=DEV)
    wd, gad, gbd = w.to(DEV), ga.to(DEV), gb.to(DEV)                                     # alive across the call
    _lib.check(e.lib.dp_debug_ws_backward(e.handle, _ptr(wd), _ptr(gad), _ptr(gbd), O, I, k, Ipad, _ptr(out), e._stream()))
    torch.cuda.synchronize()
    w64 = w.double().requires_grad_(True)
    goihw = (ga.double() + gb.double())[..., :I].permute(0, 3, 1, 2)
    (OR.standardize(w64) * goihw).sum().backward()
    r = _rel(out.cpu(), w64.grad)
    print(O, I, k, Ipad, scale, "rel", r)
    assert r <= 1e-5
