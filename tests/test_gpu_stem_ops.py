"""The bf16 engine's stem op by op against fp64, at the four image sizes that cover every tile remainder: the own
tensor-core stem forward, ConstantPad2d(1, 0) + MaxPool2d(3, 2) with its int8 argmax (forward and backward, fp32 and
bf16), and both fused stem-dgrad + masked EOT reduces (d_stem read from HBM, or rebuilt from d_pool and the argmax);
then the three stem-backward ends of the engine against each other through eot_backward and attack_grad.

Image sizes are multiples of 56, so the stem output is Ho = H / 2 = 28k.  The forward tiles are 8 x 16 output pixels,
the backward tiles 8 x 16 positions per parity class, the pooled region is indexed by H / 4.  At H = 56, 112, 168 and
224, Ho mod 8 is 4, 0, 4, 0 and Ho mod 16 is 12, 8, 4, 0.  Every output the kernels write is first filled with NaN, so
an element they leave unwritten, or add to before writing, cannot pass."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import resnetv2 as OR
from test_gpu_occlusion import _degenerate_table, _engine, _occluded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [56, 112, 168, 224]
CIN_PAD = 8   # channels per tap of the bf16 engine's stem filter (DORPATCH_CPAD unset)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


@pytest.fixture(scope="module")
def engines(oracle_params):
    made = {}

    def get(precision, H):
        if (precision, H) not in made:
            made[(precision, H)] = _engine(oracle_params, precision, img=H)
        return made[(precision, H)]
    yield get
    for e in made.values():
        e.close()


def _stem_forward(e, xb, with_w=True):
    """dp_debug_stem_forward on x [N,H,H,3] bf16 (CPU): (out [N,H/2,H/2,64] bf16, weights [64,7,7,CIN_PAD] bf16), CPU."""
    from dorpatch_b200 import _lib
    N, H = xb.shape[0], xb.shape[1]
    xd = xb.contiguous().to(DEV)
    out = _nan((N, H // 2, H // 2, 64), torch.bfloat16)
    w = _nan((64, 7, 7, CIN_PAD), torch.bfloat16) if with_w else None
    _lib.check(e.lib.dp_debug_stem_forward(e.handle, _ptr(xd), _ptr(out), _ptr(w), N, e._stream()))
    torch.cuda.synchronize()
    return out.cpu(), (w.cpu() if with_w else None)


def _stem_weights64(e, oracle_params):
    """The standardised stem weights exactly as the engine holds them, [64,3,7,7] fp64 (no host re-standardisation)."""
    _, w = _stem_forward(e, torch.zeros(1, e.img, e.img, 3, dtype=torch.bfloat16))
    assert torch.isfinite(w.float()).all() and (w[..., 3:] == 0).all()
    w64 = w[..., :3].double().permute(0, 3, 1, 2).contiguous()
    # sanity: the same weights as timm's StdConv2d standardisation rounded to bf16, within one bf16 rounding
    host = OR.standardize(oracle_params["stem.conv.weight"]).double()
    assert ((w64 - host).abs() <= 2.0 ** -8 * host.abs() + 1e-6).all()
    return w64


def _maxpool(e, x, dy=None):
    """dp_debug_maxpool on x [N,Hs,Hs,C] (CPU, the engine's dtype): (y, amax int8[, dx]) on the CPU."""
    from dorpatch_b200 import _lib
    N, Hs, _, Cc = x.shape
    xd = x.contiguous().to(DEV)
    y = _nan((N, Hs // 2, Hs // 2, Cc), x.dtype)
    amax = torch.full((N, Hs // 2, Hs // 2, Cc), -7, dtype=torch.int8, device=DEV)
    dyd = dy.contiguous().to(DEV) if dy is not None else None
    dx = _nan(x.shape, x.dtype) if dy is not None else None
    _lib.check(e.lib.dp_debug_maxpool(e.handle, _ptr(xd), _ptr(y), _ptr(amax), _ptr(dyd), _ptr(dx), N, Hs, Cc, e._stream()))
    torch.cuda.synchronize()
    return y.cpu(), amax.cpu(), (dx.cpu() if dx is not None else None)


def _maxpool_ref(x):
    """torch CPU fp64 F.max_pool2d(F.pad(x, (1,1,1,1)), 3, 2) of x [N,Hs,Hs,C]: (y NHWC fp64, argmax ky*3+kx NHWC int8,
    window-on-padding mask NHWC bool, the adjoint as a function of dy NHWC)."""
    N, Hs, _, Cc = x.shape
    xr = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    y, idx = F.max_pool2d(F.pad(xr, (1, 1, 1, 1)), 3, 2, return_indices=True)
    Ho = Hs // 2
    r, c = idx // (Hs + 2), idx % (Hs + 2)
    o = torch.arange(Ho)
    ky, kx = r - 2 * o[:, None], c - 2 * o[None, :]
    assert int(ky.min()) >= 0 and int(ky.max()) <= 2 and int(kx.min()) >= 0 and int(kx.max()) <= 2
    on_pad = (r == 0) | (c == 0)                      # the padded row / column (Hs even: only the first ones are read)
    nhwc = lambda t: t.permute(0, 2, 3, 1)            # noqa: E731

    def adjoint(dy):
        g, = torch.autograd.grad(y, xr, dy.double().permute(0, 3, 1, 2), retain_graph=True)
        return nhwc(g)
    return nhwc(y.detach()), nhwc(ky * 3 + kx).to(torch.int8), nhwc(on_pad), adjoint


GRID = torch.tensor([-1.0, -0.5, -0.0, 0.0, 0.5, 1.0])


def _pool_input(N, Hs, Cc, seed):
    """Coarse-grid activations (ties are common and exact), a quarter random; on image 0 the first two rows and columns
    (every window on the padding reads only those) are all negative in channels 0-15, all -0.0 in 16-31, negative and
    -0.0 mixed in 32-47; on image 1 only the first corner window is all negative."""
    g = torch.Generator().manual_seed(seed)
    x = GRID[torch.randint(0, len(GRID), (N, Hs, Hs, Cc), generator=g)]
    x = torch.where(torch.rand(x.shape, generator=g) < 0.25, torch.randn(x.shape, generator=g), x)
    edge = torch.zeros(Hs, Hs, dtype=torch.bool)
    edge[:2], edge[:, :2] = True, True
    neg = -(torch.rand(Hs, Hs, 16, generator=g) + 2.0 ** -6)
    x[0, :, :, 0:16] = torch.where(edge[..., None], neg, x[0, :, :, 0:16])
    x[0, :, :, 16:32] = torch.where(edge[..., None], torch.tensor(-0.0), x[0, :, :, 16:32])
    mixed = torch.where(torch.rand(Hs, Hs, 16, generator=g) < 0.5, torch.tensor(-0.0), neg)
    x[0, :, :, 32:48] = torch.where(edge[..., None], mixed, x[0, :, :, 32:48])
    if N > 1:
        x[1, :2, :2] = -(torch.rand(2, 2, Cc, generator=g) + 2.0 ** -6)
    return x


@pytest.mark.parametrize("H", SIZES)
def test_bf16_stem_forward_vs_fp64(engines, oracle_params, H):
    """The own stem convolution (7x7, stride 2, padding 3, 3 -> 64) against F.conv2d in fp64 on the same bf16 input and
    the weights the kernel reads.  Three images: random; large values (up to 64) in the outermost 3 rows and columns, where
    the padding taps matter, over a small interior; constant.  The kernel multiplies bf16 operands exactly, sums 147
    products in fp32 (error <= 147 * 2^-24 * A < 2^-16 * A, A = conv(|x|, |w|)) and rounds once to bf16 (2^-9 of the
    value), so |got - ref| <= 2^-8 |ref| + 2^-16 A elementwise.  Every output must be written (filled with NaN first)."""
    e = engines("bf16", H)
    w64 = _stem_weights64(e, oracle_params)
    g = torch.Generator().manual_seed(H)
    x = torch.rand(3, H, H, 3, generator=g) * 2 - 1
    frame = torch.zeros(H, H, dtype=torch.bool)
    frame[:3], frame[-3:], frame[:, :3], frame[:, -3:] = True, True, True, True
    x[1] = torch.where(frame[..., None], (torch.rand(H, H, 3, generator=g) * 2 - 1) * 64, x[1] * 2.0 ** -4)
    x[2] = 0.75
    xb = x.to(torch.bfloat16)
    out, _ = _stem_forward(e, xb, with_w=False)
    got = out.double().permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "unwritten outputs: %d" % int((~torch.isfinite(got)).sum())
    xd = xb.double().permute(0, 3, 1, 2)
    ref = F.conv2d(xd, w64, stride=2, padding=3)
    A = F.conv2d(xd.abs(), w64.abs(), stride=2, padding=3)
    excess = (got - ref).abs() - (2.0 ** -8 * ref.abs() + 2.0 ** -16 * A)
    bad = (excess > 0).nonzero()
    print("stem forward H=%d: max |got-ref| / max |ref| %.2e, violations %d"
          % (H, float((got - ref).abs().max() / ref.abs().max()), len(bad)))
    assert len(bad) == 0, ("[n, k, oy, ox]", bad[:8].tolist())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("H", SIZES)
def test_maxpool_fwd_bwd_vs_fp64(engines, precision, H):
    """Pad + max-pool at Hs = H / 2, C = 64, against torch CPU fp64 on the same (dtype-rounded) values.  The pooled
    values are selections, so y matches bit for bit, sign of zero included (the padding is +0.0 and comes first in every
    window that reads it, so it beats -0.0), and the argmax ky*3+kx matches exactly (first maximum in row-major window
    order).  dy is drawn from multiples of 1/64 in [-2, 2], so a <= 4-term sum is exact in fp32: fp32 dx is exact, bf16
    dx within its one rounding, 2^-8 |ref|.  Windows whose maximum is the padding send nothing back: exactly zero dx."""
    e = engines(precision, 56)                       # the hook takes Hs and C: one small engine per dtype
    dt = torch.bfloat16 if precision == "bf16" else torch.float32
    Hs, N, Cc = H // 2, 2, 64
    x = _pool_input(N, Hs, Cc, seed=H).to(dt)
    dy = (torch.randint(-128, 129, (N, Hs // 2, Hs // 2, Cc), generator=torch.Generator().manual_seed(H + 1)) / 64.0).to(dt)
    y, amax, dx = _maxpool(e, x, dy)
    y_ref, amax_ref, on_pad, adjoint = _maxpool_ref(x)
    bits = torch.int16 if dt == torch.bfloat16 else torch.int32
    assert on_pad.any() and (y_ref[on_pad] == 0).any() and (x == 0).any()
    nbad = int((y.view(bits) != y_ref.to(dt).view(bits)).sum())
    assert nbad == 0, "max-pool values differ (bits) at %d elements" % nbad
    nbad = int((amax != amax_ref).sum())
    assert nbad == 0, "argmax differs at %d elements" % nbad
    dx_ref = adjoint(dy)
    assert torch.isfinite(dx.float()).all()
    err = (dx.double() - dx_ref).abs()
    tol = 2.0 ** -8 * dx_ref.abs() if dt == torch.bfloat16 else torch.zeros_like(dx_ref)
    assert (err <= tol).all(), "dx: %d elements off, max %.3g" % (int((err > tol).sum()), float(err.max()))
    _, _, dx_pad = _maxpool(e, x, torch.where(on_pad, dy, torch.zeros_like(dy)))
    assert int(on_pad.sum()) > 0 and (dx_pad == 0).all(), "gradient flowed from windows whose maximum is the padding"


@pytest.mark.parametrize("H", SIZES)
def test_bf16_fused_stem_bwd_reduces_vs_fp64(engines, oracle_params, H):
    """Both fused stem-dgrad + masked EOT reduces on the degenerate rectangle tables, two images, so the second image's
    samples start mid-launch.  d_pool (bf16) and the argmax come from the max-pool hook on a random stem output; its
    backward gives d_stem.  Reference: the fp64 max-pool adjoint rounded to bf16 (the engine's d_stem is bf16), then
    conv_transpose2d in fp64 with the engine's weights, then 2 * sum over samples of keep.  Both sides multiply exact
    bf16 products; the kernel sums in fp32: relative L2 <= 1e-5, max abs <= 1e-4 of the max.  The PoolPatch reduce
    rebuilds d_stem in shared memory with the same fp32 sums and one rounding, so it matches the d_stem reduce bit for
    bit.  G is filled with NaN first and must be fully written."""
    from dorpatch_b200 import _lib
    e = engines("bf16", H)
    w64 = _stem_weights64(e, oracle_params)
    rects = _degenerate_table(H, n_random=1)                     # 20 samples: B = 2, S = 10
    B, S = 2, len(rects) // 2
    N, hs, hp = B * S, H // 2, H // 4
    g = torch.Generator().manual_seed(100 + H)
    x_stem = torch.randn(N, hs, hs, 64, generator=g).to(torch.bfloat16)
    dpool = ((torch.rand(N, hp, hp, 64, generator=g) * 2 - 1) * 1e-2).to(torch.bfloat16)
    _, amax, dstem = _maxpool(e, x_stem, dpool)
    _, amax_ref, _, adjoint = _maxpool_ref(x_stem)
    assert torch.equal(amax, amax_ref)
    dstem_ref = adjoint(dpool).to(torch.bfloat16)
    rects_c = np.ascontiguousarray(rects, np.int16)
    Gs = []
    for name in ("dy", "pool"):
        G = _nan((B, 3, H, H), torch.float32)
        if name == "dy":
            src = dstem.to(DEV)
            _lib.check(e.lib.dp_debug_stem_bwd_reduce(e.handle, _ptr(src), C.c_void_p(rects_c.ctypes.data), B, S, _ptr(G),
                                                      e._stream()))
        else:
            src, am = dpool.to(DEV), amax.to(DEV)
            _lib.check(e.lib.dp_debug_stem_bwd_pool_reduce(e.handle, _ptr(src), _ptr(am), C.c_void_p(rects_c.ctypes.data),
                                                           B, S, _ptr(G), e._stream()))
        torch.cuda.synchronize()
        G = G.cpu()
        assert torch.isfinite(G).all(), "%s: %d elements of G not written" % (name, int((~torch.isfinite(G)).sum()))
        Gs.append(G)
    dX = F.conv_transpose2d(dstem_ref.double().permute(0, 3, 1, 2), w64, stride=2, padding=3, output_padding=1)
    keep = torch.from_numpy(~_occluded(rects, H)).double()[:, None]
    ref = 2.0 * (dX * keep).reshape(B, S, 3, H, H).sum(1)
    got = Gs[0].double()
    rel = float((got - ref).norm() / ref.norm())
    mx = float((got - ref).abs().max() / ref.abs().max())
    nd = int((Gs[0] != Gs[1]).sum())
    print("stem bwd reduces H=%d: rel L2 %.2e, max abs / max %.2e; pool vs dy: %d elements differ" % (H, rel, mx, nd))
    assert rel <= 1e-5 and mx <= 1e-4, (rel, mx)
    assert nd == 0, "PoolPatch differs from DyPatch at %d elements, max %.3g" % (nd, float((Gs[0] - Gs[1]).abs().max()))


ENDS = {"cudnn": {"DORPATCH_STEM_BWD": "cudnn"}, "default": {}, "pool": {"DORPATCH_POOL_BWD": "fused"}}
CHUNKINGS = {        # (B, S, chunk)
    "two-lanes": (2, 4, 4),        # each chunk one whole image, on two lanes, both held from the forward
    "straddle": (2, 9, 4),         # images straddle chunks: one stream, accumulated across chunks
    "recompute": (4, 2, 2),        # whole images on two lanes, four chunks: two are recomputed in the backward
}


@pytest.mark.parametrize("chunking", list(CHUNKINGS))
def test_bf16_stem_backward_ends_agree(oracle_params, chunking):
    """One bf16 engine at H = 112 per stem-backward end: cuDNN's dgrad + reduce (DORPATCH_STEM_BWD=cudnn), the fused
    dgrad + reduce (default), and that plus the fused max-pool backward (DORPATCH_POOL_BWD=fused).  eot_forward +
    eot_backward (image gradient filled with NaN first) and attack_grad (G filled with NaN first) at three chunkings.
    All values finite; logits and losses identical; default and pool identical bit for bit (the rebuilt d_stem patch
    holds maxpool_bwd_kernel's values); each fused end against cuDNN's, which rounds every sample's input gradient to
    bf16 before the reduce: cosine >= 0.9999, relative L2 <= 1e-2."""
    H = 112
    B, S, chunk = CHUNKINGS[chunking]
    rects = _degenerate_table(H, n_random=0)[:B * S].reshape(B, S, 4, 4)
    g = torch.Generator().manual_seed(21)
    x, m, p = torch.rand(B, 3, H, H, generator=g), torch.rand(B, 1, H, H, generator=g), torch.rand(B, 3, H, H, generator=g)
    dlog = torch.randn(B * S, 1000, generator=torch.Generator().manual_seed(22))
    y = np.array([17, 400, 3, 999][:B])
    res = {}
    for end, env in ENDS.items():
        e = _engine(oracle_params, "bf16", chunk=chunk, max_images=B, **env)
        try:
            dl = dlog.to(DEV)
            logits = e.eot_forward(x.to(DEV), S, rects)           # the image is a temporary the engine must keep
            Ge = _nan((B, 3, H, H), torch.float32)                # the first allocation after it, of the image's size
            e.eot_backward(dl, out=Ge)
            torch.cuda.synchronize()
            Ge, logits = Ge.cpu(), logits.cpu()
            Ga = _nan((B, 3, H, H), torch.float32)
            r = e.attack_grad(x.to(DEV), m.to(DEV), p.to(DEV), rects, y, [True, False, True, False][:B], 0.1, 4.0, 1, Ga)
            torch.cuda.synchronize()
            res[end] = {"logits": logits, "loss": torch.from_numpy(r["loss_adv"].copy()), "eot": Ge, "attack": Ga.cpu()}
        finally:
            e.close()
    for end in ENDS:
        for k in ("eot", "attack"):
            G = res[end][k]
            assert torch.isfinite(G).all(), "%s %s: %d non-finite elements" % (end, k, int((~torch.isfinite(G)).sum()))
        assert torch.equal(res[end]["logits"], res["default"]["logits"]) and torch.equal(res[end]["loss"], res["default"]["loss"])
    for k in ("eot", "attack"):
        ref = res["cudnn"][k].double()
        assert ref.abs().sum() > 0
        for end in ("default", "pool"):
            got = res[end][k].double()
            cos = float((got * ref).sum() / (got.norm() * ref.norm()))
            rel = float((got - ref).norm() / ref.norm())
            print("%s %s %s vs cudnn: cos %.7f rel %.2e" % (chunking, k, end, cos, rel))
            assert cos >= 0.9999 and rel <= 1e-2, (k, end, cos, rel)
        d = (res["pool"][k] - res["default"][k]).abs()
        assert torch.equal(res["pool"][k], res["default"][k]), (k, "pool vs default: max %.3g" % float(d.max()))


def test_eot_backward_keeps_and_checks_the_image(oracle_params):
    """eot_backward recomputes the chunks the engine no longer holds from the image given to eot_forward, so the engine
    keeps that tensor alive (a temporary's memory would otherwise go to the next allocation, such as the gradient), and
    refuses a backward after an in-place change of the image or into a buffer that shares its memory."""
    import weakref
    H, B, S = 112, 2, 9
    rects = _degenerate_table(H, n_random=0)[:B * S].reshape(B, S, 4, 4)
    e = _engine(oracle_params, "bf16", chunk=4, max_images=B)
    try:
        img = torch.rand(B, 3, H, H, generator=torch.Generator().manual_seed(31)).to(DEV)
        alive = weakref.ref(img)
        dl = torch.randn(B * S, 1000, generator=torch.Generator().manual_seed(32)).to(DEV)
        e.eot_forward(img, S, rects)
        del img
        assert alive() is not None
        g = e.eot_backward(dl)
        assert torch.isfinite(g).all()
        with pytest.raises(ValueError, match="shares memory"):
            e.eot_backward(dl, out=alive())
        alive().mul_(0.5)
        with pytest.raises(RuntimeError, match="modified in place"):
            e.eot_backward(dl)
        with pytest.raises(RuntimeError, match="modified in place"):
            e.eot_backward_params(dl, ["head.fc.bias"], [torch.empty(1000, device=DEV)])
    finally:
        e.close()
