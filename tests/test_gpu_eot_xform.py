"""Affine / colour EOT in the differentiable classifier (dp_eot_forward_xform, Engine.eot_forward(xforms=...),
ops.eot_logits(xforms=...)): against the torch restatement of the transform with the oracle classifier under autograd,
against dp_attack_grad's affine path (the arithmetic generate(eot_affine=..., eot_colour=...) optimises), resident vs
recomputed chunks, the identity transform, the unchanged no-transform path, and the errors.

The warp adjoint (reduce_affine_kernel) adds with fp32 atomics, so gradients after a transformed forward are compared
with a relative L2 bound instead of bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dorpatch_b200 import _lib
from dorpatch_b200 import eot as PE
from dorpatch_b200 import masks as PM
from oracle import attack as OA
from oracle import eot as OE
from oracle import resnetv2 as OR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRECISIONS = ["fp32", "tf32", "bf16"]


def _rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _rects(H, B, S, seed, dropout=2):
    table = PM.universe(H, dropout)
    idx = np.random.RandomState(seed).randint(0, table.shape[0], (B, S))
    return table, idx, PM.gather(table, idx)


def _xforms(B, S, seed, affine=0.1, colour=0.1):
    return PE.sample(np.random.RandomState(seed), B, S, affine, colour)


def _cw(logits, y, targeted, confidence, w):
    """Per-sample CW loss and d(w * sum_n cw_n)/d logits as cw_kernel forms them (attack.py:16-23; no top-2 ties)."""
    N, K = logits.shape
    n = torch.arange(N, device=logits.device)
    real = logits[n, y]
    oi = logits.masked_fill(F.one_hot(y, K).bool(), float("-inf")).argmax(1)
    other = logits[n, oi]
    pre = confidence + torch.where(targeted, other - real, real - other)
    live = pre >= 0
    d = torch.zeros_like(logits)
    sgn = torch.where(targeted, -1.0, 1.0).to(logits.device) * w
    d[n, y] = torch.where(live, sgn, 0.0)
    d[n, oi] = torch.where(live, -sgn, 0.0)
    return pre.clamp(min=0), d


@pytest.fixture(scope="module")
def engines(oracle_params):
    """Engines of this module, freed at its end (the 224 px ones are large)."""
    from dorpatch_b200.engine import Engine
    made = {}

    def get(img, precision, chunk, max_images):
        key = (img, precision, chunk, max_images)
        if key not in made:
            e = Engine(img=img, precision=precision, chunk=chunk, max_images=max_images, autotune=False)
            e.load_state_dict(oracle_params)
            made[key] = e
        return made[key]
    yield get
    for e in made.values():
        e.close()
    torch.cuda.empty_cache()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ---------------------------------------------------------------------------------------------------------------
def _kernel_warp(adv, xf):
    """The warp as expand_affine_kernel computes its sampling points ((2w+1)/W - 1 per pixel, then theta, then
    ((x + 1) W - 1) / 2, clamped to the border), in torch and differentiable: [B,3,H,W], [B,S,8] -> [B,S,3,H,W].
    F.affine_grid builds its base grid from a linspace instead, which puts the points ~1e-6 pixel elsewhere."""
    B, _, H, W = adv.shape
    S = xf.shape[1]
    h, w = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    xn, yn = (2 * w + 1) / W - 1, (2 * h + 1) / H - 1
    out = []
    for b in range(B):
        pl = adv[b].reshape(3, -1)
        for s in range(S):
            t = torch.from_numpy(xf[b, s])
            fx = (((t[0] * xn + t[1] * yn + t[2] + 1) * W - 1) * 0.5).clamp(0, W - 1)
            fy = (((t[3] * xn + t[4] * yn + t[5] + 1) * H - 1) * 0.5).clamp(0, H - 1)
            x0, y0 = fx.floor().long(), fy.floor().long()
            ax, ay = fx - x0, fy - y0
            x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)
            ox, oy = (x0 + 1 < W).float(), (y0 + 1 < H).float()
            v = sum(pl[:, (yy * W + xx).reshape(-1)] * wt.reshape(-1) for yy, xx, wt in (
                (y0, x0, (1 - ax) * (1 - ay)), (y0, x1, ox * ax * (1 - ay)),
                (y1, x0, (1 - ax) * oy * ay), (y1, x1, ox * ax * oy * ay)))
            out.append(torch.clamp(t[6] * (v - 0.5) + 0.5 + t[7], 0.0, 1.0).reshape(3, H, W))
    return torch.stack(out).reshape(B, S, 3, H, W)


@pytest.mark.parametrize("H", [112, 224])
@pytest.mark.parametrize("image,warp", [("smooth", "oracle"), ("noise", "kernel_points")])
def test_xform_cross_entropy_vs_oracle(engines, oracle_params, H, image, warp):
    """fp32, cross-entropy over transformed (affine 0.1, colour 0.1) and occluded samples against torch autograd
    through a torch warp and the oracle classifier: logits within 2e-3, input-gradient cosine >= 0.999.

    smooth / oracle: a low-frequency image (bilinear upsampling of an H/8 noise image) through oracle/eot.py's
    F.affine_grid + F.grid_sample restatement.  Measured on an H100: cosine 0.99983 (112 px), 0.99960 (224 px).
    noise / kernel_points: pixel noise through the same bilinear warp at the kernel's sampling points
    (_kernel_warp).  Measured: 0.99992, 0.99981.  Logits within 2.8e-5 in all four.
    Pixel noise through grid_sample gives 0.9986 and 0.9976: grid_sample samples ~1e-6 pixel away from the kernel,
    which on pixel noise moves the classifier's input by up to 2e-5 and flips ReLU gates and max-pool choices of the
    random-init classifier; the identity test below shows the same effect without any oracle."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    B, S = 2, 3
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    net.adopt_engine(engines(H, "fp32", 4, 4))
    img = _rand((B, 3, H, H), 61)
    if image == "smooth":
        img = F.interpolate(_rand((B, 3, H // 8, H // 8), 64), size=(H, H), mode="bilinear", align_corners=False)
    table, idx, rects = _rects(H, B, S, 62)
    xf = _xforms(B, S, 63)
    y = torch.tensor([5, 321]).repeat_interleave(S)
    xd = img.to(DEV).requires_grad_(True)
    logits = eot_logits(net, xd, rects, S, xforms=xf)
    F.cross_entropy(logits, y.to(DEV)).backward()
    keep = torch.from_numpy(PM.to_bool(table, H)[idx])                      # [B,S,1,H,W]
    xr = img.clone().requires_grad_(True)
    warped = OE.apply(xr, xf) if warp == "oracle" else _kernel_warp(xr, xf)
    ref = OR.forward(oracle_params, OA.occlude(warped, keep).reshape(B * S, 3, H, H))
    F.cross_entropy(ref, y).backward()
    err = (logits.detach().cpu() - ref.detach()).abs().max().item()
    cos = _cos(xd.grad.cpu(), xr.grad)
    print("H", H, image, warp, "logit err", err, "grad cos", cos)
    assert err <= 2e-3
    assert cos >= 0.999


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("B,S", [(1, 128), (4, 32)])
def test_xform_cw_backward_matches_attack_grad(engines, precision, B, S):
    """The CW gradient formed in torch from eot_forward(xforms=...) and pushed through eot_backward against
    dp_attack_grad's grad_adv (stage 1) for the same transforms and rectangles at 224 px: argmax = dp_attack_grad's
    preds bit for bit, losses within 1e-6, gradients within 1e-5 relative L2 (both sum with atomics)."""
    H = 224
    e = engines(H, precision, 64, 4)
    x, m, p = _rand((B, 3, H, H), 71).to(DEV), _rand((B, 1, H, H), 72).to(DEV), _rand((B, 3, H, H), 73).to(DEV)
    _, _, rects = _rects(H, B, S, 74)
    xf = _xforms(B, S, 75, affine=0.5, colour=0.5)
    y = np.array([17, 400, 3, 999][:B])
    targeted = np.array([True, False, True, False][:B])
    G = torch.zeros(B, 3, H, H, device=DEV)
    r = e.attack_grad(x, m, p, rects, y, targeted, 0.1, 4.0, 1, G, xforms=xf)
    adv, _, _ = e.paste(x, m, p, 4.0)
    logits = e.eot_forward(adv, S, rects, xforms=xf)
    top2 = logits.topk(2, dim=1).values
    assert bool((top2[:, 0] > top2[:, 1]).all()), "inputs with a top-2 tie: pick other seeds"
    assert np.array_equal(logits.argmax(1).cpu().numpy(), r["preds"].reshape(-1))
    yy = torch.from_numpy(np.repeat(y, S)).to(DEV)
    tt = torch.from_numpy(np.repeat(targeted, S)).to(DEV)
    loss, d = _cw(logits, yy, tt, 0.1, 1.0 / S)
    assert np.abs(loss.cpu().numpy() - r["loss_adv"].reshape(-1)).max() <= 1e-6
    g = e.eot_backward(d)
    torch.cuda.synchronize()
    rel = _rel_l2(g, G)
    print(precision, B, S, "grad rel L2", rel)
    assert rel <= 1e-5


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_xform_resident_and_recomputed_chunks(engines, precision):
    """Chunk 4, B = 5 images x S = 4 transformed samples (5 chunks; the backward recomputes three): the logits are bit
    for bit those of five one-image calls (one chunk each, nothing recomputed), and so is the gradient within 1e-5
    relative L2; a second backward of the same forward agrees to the same bound.  With images split across chunks
    (S = 3) the gradient is the sum of the backwards of dlogits restricted to one chunk at a time."""
    H = 112
    e = engines(H, precision, 4, 5)
    B, S = 5, 4
    img = _rand((B, 3, H, H), 81).to(DEV)
    _, _, rects = _rects(H, B, S, 82)
    xf = _xforms(B, S, 83, affine=0.5, colour=0.5)
    dl = (_rand((B * S, 1000), 84) - 0.5).to(DEV)
    logits = e.eot_forward(img, S, rects, xforms=xf)
    g = e.eot_backward(dl)
    g2 = e.eot_backward(dl)
    torch.cuda.synchronize()
    assert _rel_l2(g2, g) <= 1e-5
    lparts, gparts = [], []
    for b in range(B):
        lparts.append(e.eot_forward(img[b:b + 1].contiguous(), S, rects[b:b + 1], xforms=xf[b:b + 1]))
        gparts.append(e.eot_backward(dl[b * S:(b + 1) * S].contiguous()))
    assert torch.equal(logits, torch.cat(lparts))
    rel = _rel_l2(g, torch.cat(gparts))
    print(precision, "recomputed vs resident rel L2", rel)
    assert rel <= 1e-5

    B, S = 5, 3                                            # 15 samples over chunks of 4: images span chunks
    _, _, rects = _rects(H, B, S, 85)
    xf = _xforms(B, S, 86, affine=0.5, colour=0.5)
    dl = (_rand((B * S, 1000), 87) - 0.5).to(DEV)
    e.eot_forward(img, S, rects, xforms=xf)
    g = e.eot_backward(dl)
    acc = None
    for n0 in range(0, B * S, 4):
        d = torch.zeros_like(dl)
        d[n0:n0 + 4] = dl[n0:n0 + 4]
        gc = e.eot_backward(d)
        acc = gc if acc is None else acc + gc
    torch.cuda.synchronize()
    assert _rel_l2(acc, g) <= 1e-5


@pytest.mark.parametrize("precision", ["fp32"])
def test_identity_transform_matches_plain_path(engines, precision):
    """theta = identity, contrast 1, brightness 0: the warp samples every pixel at its own centre up to ~1e-6 pixel of
    float rounding, so the logits are within 1e-4 of the xforms=None path (measured on an H100: 2.5e-5) and the
    cross-entropy input gradient has cosine >= 0.9995 with it.  Measured: 0.99981 on this pixel-noise image; the
    rounding moves the input by up to ~1e-6 and flips a few ReLU gates / max-pool choices of the random-init
    classifier (a low-frequency image gives 0.99993)."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, B, S = 112, 2, 4
    net = ResNetV2(seed=0)
    e = engines(H, precision, 4, 4)
    net.adopt_engine(e)
    img = _rand((B, 3, H, H), 91).to(DEV)
    _, _, rects = _rects(H, B, S, 92)
    xf = np.tile(np.array([1, 0, 0, 0, 1, 0, 1, 0], np.float32), (B, S, 1))
    y = torch.tensor([7, 600], device=DEV).repeat_interleave(S)
    x0 = img.clone().requires_grad_(True)
    l0 = eot_logits(net, x0, rects, S)
    F.cross_entropy(l0, y).backward()
    x1 = img.clone().requires_grad_(True)
    l1 = eot_logits(net, x1, rects, S, xforms=torch.from_numpy(xf))
    F.cross_entropy(l1, y).backward()
    err = (l1 - l0).abs().max().item()
    cos = _cos(x1.grad, x0.grad)
    print("identity: logit err", err, "grad cos", cos)
    assert err <= 1e-4
    assert cos >= 0.9995


@pytest.mark.parametrize("precision", PRECISIONS)
def test_no_transform_path_unchanged(engines, precision):
    """xforms=None is dp_eot_forward + dp_eot_backward bit for bit (logits and gradient), through Engine and through
    eot_logits, including right after a transformed forward / backward on the same engine."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, B, S = 112, 3, 4                                    # 12 samples over chunks of 4: one chunk recomputed
    e = engines(H, precision, 4, 4)
    net = ResNetV2(seed=0)
    net.adopt_engine(e)
    img = _rand((B, 3, H, H), 101).to(DEV)
    _, _, rects = _rects(H, B, S, 102)
    dl = (_rand((B * S, 1000), 103) - 0.5).to(DEV)
    rh = np.ascontiguousarray(rects.reshape(B * S, 4, 4), np.int16)

    def raw():
        logits = torch.empty(B * S, 1000, device=DEV)
        g = torch.empty_like(img)
        _lib.check(e.lib.dp_eot_forward(e.handle, _ptr(img), B, S, C.c_void_p(rh.ctypes.data), _ptr(logits),
                                        e._stream()))
        _lib.check(e.lib.dp_eot_backward(e.handle, _ptr(dl), _ptr(g), e._stream()))
        return logits, g

    l_ref, g_ref = raw()
    l_eng = e.eot_forward(img, S, rects, xforms=None)
    g_eng = e.eot_backward(dl)
    assert torch.equal(l_eng, l_ref) and torch.equal(g_eng, g_ref)
    e.eot_forward(img, S, rects, xforms=_xforms(B, S, 104))
    e.eot_backward(dl)
    l_after, g_after = raw()
    assert torch.equal(l_after, l_ref) and torch.equal(g_after, g_ref)
    x = img.clone().requires_grad_(True)
    logits = eot_logits(net, x, rects, S, xforms=None)
    (logits * dl).sum().backward()
    assert torch.equal(logits.detach(), l_ref)
    assert torch.equal(x.grad, g_ref)


def test_xform_errors(engines):
    """A backward after dp_predict raises "stale forward"; double backward raises; non-finite transforms, B above
    max_images and a null image are refused with a message; a refused forward leaves the last one differentiable."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, B, S = 112, 2, 3
    e = engines(H, "fp32", 4, 4)
    net = ResNetV2(seed=0)
    net.adopt_engine(e)
    img = _rand((B, 3, H, H), 111).to(DEV)
    xf = _xforms(B, S, 112)
    y = torch.tensor([1, 2], device=DEV).repeat_interleave(S)

    x = img.clone().requires_grad_(True)
    loss = F.cross_entropy(eot_logits(net, x, None, S, xforms=xf), y)
    e.predict(img)
    with pytest.raises(RuntimeError, match="stale forward"):
        loss.backward()
    assert x.grad is None

    x = img.clone().requires_grad_(True)
    loss = F.cross_entropy(eot_logits(net, x, None, S, xforms=xf), y)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(loss, x, create_graph=True)

    dl = (_rand((B * S, 1000), 113) - 0.5).to(DEV)
    e.eot_forward(img, S, None, xforms=xf)
    g = e.eot_backward(dl)
    for bad in (np.nan, np.inf, -np.inf):
        xb = xf.copy()
        xb[1, 2, 6] = bad
        with pytest.raises(RuntimeError, match="non-finite"):
            e.eot_forward(img, S, None, xforms=xb)
        with pytest.raises(RuntimeError, match="non-finite"):
            eot_logits(net, img.clone().requires_grad_(True), None, S, xforms=xb)
    big = _rand((5, 3, H, H), 114).to(DEV)
    with pytest.raises(RuntimeError, match="max_images"):
        e.eot_forward(big, S, None, xforms=_xforms(5, S, 115))
    logits = torch.empty(B * S, 1000, device=DEV)
    xh = np.ascontiguousarray(xf.reshape(-1, 8))
    rc = e.lib.dp_eot_forward_xform(e.handle, None, B, S, None, C.c_void_p(xh.ctypes.data), _ptr(logits), e._stream())
    assert rc != 0 and b"null pointer" in e.lib.dp_last_error()
    g2 = e.eot_backward(dl)
    torch.cuda.synchronize()
    assert _rel_l2(g2, g) <= 1e-5
