"""The occlusion table through every kernel that reads it: degenerate rectangle tables (empty, one pixel, full image,
touching each edge, overlapping, all four slots) through K1 at every input layout the engines use and through the
fused bf16 stem-dgrad + masked EOT reduce; and the two fused stem-backward variants (dY copied, or rebuilt from d_pool
and the max-pool argmax) against each other."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import resnetv2 as OR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H = 112


def _degenerate_table(H, n_random=56, seed=0):
    """[n,4,4] int16 tables, one sample per row, four {r0, r1, c0, c1} rectangles per sample."""
    E = [0, 0, 0, 0]
    cases = [
        [E, E, E, E],                                              # no occlusion
        [[5, 5, 0, H], E, E, E],                                   # r0 == r1
        [E, [0, H, 7, 7], E, E],                                   # c0 == c1
        [E, E, [30, 10, 0, H], E],                                 # r1 < r0
        [E, E, E, [0, H, 40, 20]],                                 # c1 < c0
        [[17, 18, 23, 24], E, E, E],                               # one pixel
        [E, E, E, [H - 1, H, H - 1, H]],                           # one pixel in the last corner
        [[0, 1, 0, 1], E, [50, 51, 61, 62], E],                    # one pixel in the first corner, one inside
        [[0, H, 0, H], E, E, E],                                   # the whole image
        [[0, 9, 30, 60], E, E, E],                                 # top edge
        [[H - 9, H, 30, 60], E, E, E],                             # bottom edge
        [[40, 70, 0, 11], E, E, E],                                # left edge
        [[40, 70, H - 11, H], E, E, E],                            # right edge
        [[0, H, 0, 3], [0, 3, 0, H], [0, H, H - 3, H], [H - 3, H, 0, H]],   # a frame: all four edges, four slots
        [[10, 50, 10, 50], [30, 70, 30, 70], E, E],                # overlapping
        [[10, 50, 10, 50], [10, 50, 10, 50], [20, 30, 20, 30], E], # repeated, and one inside another
        [[3, 20, 5, 9], [60, 61, 0, H], [0, H, 77, 78], [90, 112, 100, 101]],  # all four slots, thin strips
        [[8, 16, 8, 16], [16, 24, 16, 24], [24, 32, 24, 32], [32, 40, 32, 40]],  # all four, on tile / chunk borders
        [[5, 5, 5, 5], [9, 3, 0, H], [0, H, 9, 3], [20, 21, 20, 21]],   # three empty kinds beside one pixel
    ]
    t = np.array(cases, np.int16)
    rng = np.random.RandomState(seed)
    r = rng.randint(0, H + 1, (n_random, 4, 4))
    r[:, :, [0, 1]] = np.sort(r[:, :, [0, 1]], -1)
    r[:, :, [2, 3]] = np.sort(r[:, :, [2, 3]], -1)
    r[::7, 1, [0, 1]] = r[::7, 1, [1, 0]]                         # some rows reversed (empty)
    r[3::7, 2, 3] = r[3::7, 2, 2]                                 # some zero-width
    return np.concatenate([t, r.astype(np.int16)])


def _occluded(rects, H):
    """[n,H,H] bool: the union of each sample's (half-open) rectangles."""
    pos = np.arange(H)
    occ = np.zeros((len(rects), H, H), bool)
    for s in range(4):
        r0, r1, c0, c1 = (rects[:, s, q].astype(np.int64)[:, None] for q in range(4))
        occ |= ((pos >= r0) & (pos < r1))[:, :, None] & ((pos >= c0) & (pos < c1))[:, None, :]
    return occ


def _occlude_normalise_nhwc(img, rects):
    """(occlude(img, rects) - 0.5) / 0.5 as [n,H,W,3] float32: occluded pixels are zero."""
    z = ((img - np.float32(0.5)) / np.float32(0.5)).transpose(1, 2, 0)
    return np.where(_occluded(rects, img.shape[-1])[..., None], np.float32(0.0), z[None])


@contextlib.contextmanager
def _env(**kv):
    """Set DORPATCH_* variables while an engine is created (they are read once, at create)."""
    saved = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _engine(oracle_params, precision, img=H, chunk=8, max_images=2, **env):
    from dorpatch_b200.engine import Engine
    with _env(**env):
        e = Engine(img=img, precision=precision, chunk=chunk, max_images=max_images, autotune=False)
    e.load_state_dict(oracle_params)
    return e


LAYOUTS = [   # (precision, environment at create, channels per pixel of the network input)
    ("bf16", {}, 3),
    ("bf16", {"DORPATCH_STEM": "cudnn"}, 8),
    ("bf16", {"DORPATCH_STEM": "cudnn", "DORPATCH_CPAD": "4"}, 4),
    ("fp32", {}, 4),
    ("fp32", {"DORPATCH_CPAD": "8"}, 8),
]


@pytest.mark.parametrize("precision,env,cp", LAYOUTS, ids=["bf16-c3", "bf16-c8", "bf16-c4", "fp32-c4", "fp32-c8"])
def test_expand_degenerate_rectangles(oracle_params, precision, env, cp):
    """K1 (dp_expand) on the degenerate tables, bit for bit against numpy: fp32 exact, bf16 the rounding of the fp32
    result.  Three launch shapes: the default (a sample group's rectangles cached in shared memory), one sample group
    of all 75 samples (read from global memory), and 16-byte stores only."""
    e = _engine(oracle_params, precision, **env)
    try:
        assert e.c_pad == cp
        rects = _degenerate_table(H)
        img = torch.rand(1, 3, H, H, generator=torch.Generator().manual_seed(5))
        ref = torch.from_numpy(_occlude_normalise_nhwc(img[0].numpy(), rects))
        if precision == "bf16":
            ref = ref.bfloat16().float()
        for rows, sg, mode in ((0, 0, 0), (0, 1, 0), (0, 0, 1)):
            e.lib.dp_debug_k1_tuning(rows, sg, mode)
            got = e.expand(img.to(DEV), len(rects), rects).float().cpu()
            torch.cuda.synchronize()
            assert got.shape == (len(rects), H, H, cp) and (got[..., 3:] == 0).all()
            bad = (got[..., :3] != ref).any(-1).any(-1).any(-1).nonzero().flatten().tolist()
            assert not bad, ("launch shape", rows, sg, mode, "samples", bad[:8])
    finally:
        e.lib.dp_debug_k1_tuning(0, 0, 0)
        e.close()


def test_bf16_stem_bwd_reduce_degenerate_rectangles(oracle_params):
    """The fused stem dgrad + masked EOT reduce on the degenerate tables against torch fp32 conv_transpose2d on the same
    bf16 operands, within the bounds of test_bf16_stem_bwd_reduce_vs_torch_fp32 (only the summation order differs).
    Two images, so the second image's samples start mid-launch."""
    from dorpatch_b200 import _lib
    e = _engine(oracle_params, "bf16")
    try:
        rects = _degenerate_table(H, n_random=59)                  # 78 samples: B = 2, S = 39
        B, S = 2, len(rects) // 2
        N, hs = B * S, H // 2
        dY = (torch.rand((N, hs, hs, 64), generator=torch.Generator().manual_seed(13)) * 2e-2 - 1e-2).to(torch.bfloat16)
        G = torch.empty(B, 3, H, H, device=DEV)
        dYd = dY.to(DEV)
        rects_c = np.ascontiguousarray(rects, np.int16)
        _lib.check(e.lib.dp_debug_stem_bwd_reduce(e.handle, C.c_void_p(dYd.data_ptr()), C.c_void_p(rects_c.ctypes.data),
                                                  B, S, C.c_void_p(G.data_ptr()), e._stream()))
        torch.cuda.synchronize()
    finally:
        e.close()
    w = OR.standardize(oracle_params["stem.conv.weight"]).to(torch.bfloat16).float()
    dX = F.conv_transpose2d(dY.float().permute(0, 3, 1, 2), w, stride=2, padding=3, output_padding=1)
    ref = 2.0 * (dX * torch.from_numpy(~_occluded(rects, H)).float()[:, None]).reshape(B, S, 3, H, H).sum(1)
    got = G.cpu()
    rel = float((got - ref).norm() / ref.norm())
    mx = float((got - ref).abs().max() / ref.abs().max())
    print("stem_bwd_reduce, degenerate rectangles: rel L2 %.2e, max abs / max %.2e" % (rel, mx))
    assert rel <= 1e-5 and mx <= 1e-4, (rel, mx)


def _default_and_pool(oracle_params, call):
    """The image gradient of one call on two bf16 engines with the same weights and inputs: the default stem backward,
    and DORPATCH_POOL_BWD=fused (the d_stem patch rebuilt from d_pool and the saved argmax inside the fused kernel)."""
    B, S = 2, 9                                                    # chunk 4: images straddle chunks
    rects = _degenerate_table(H, n_random=0)[:B * S].reshape(B, S, 4, 4)
    g = torch.Generator().manual_seed(21)
    x, m, p = torch.rand(B, 3, H, H, generator=g), torch.rand(B, 1, H, H, generator=g), torch.rand(B, 3, H, H, generator=g)
    out = []
    for env in ({}, {"DORPATCH_POOL_BWD": "fused"}):
        e = _engine(oracle_params, "bf16", chunk=4, **env)
        try:
            if call == "attack_grad":
                G = torch.zeros(B, 3, H, H, device=DEV)
                r = e.attack_grad(x.to(DEV), m.to(DEV), p.to(DEV), rects, np.array([17, 400]), [True, False], 0.1, 4.0, 1, G)
                side = r["loss_adv"].copy()
            else:
                logits = e.eot_forward(x.to(DEV), S, rects)
                G = e.eot_backward(torch.randn(logits.shape, generator=torch.Generator().manual_seed(22)).to(DEV))
                side = logits.cpu().numpy()
            torch.cuda.synchronize()
            out.append((G.cpu(), side))
        finally:
            e.close()
    (ga, sa), (gb, sb) = out
    assert np.array_equal(sa, sb) and ga.abs().sum() > 0
    return ga, gb


def test_bf16_pool_fused_stem_backward_matches_default_attack_grad(oracle_params):
    """The rebuilt d_stem patch holds the bf16 values maxpool_bwd_kernel writes, so dp_attack_grad's (stage 1) image
    gradient is bit-identical with and without DORPATCH_POOL_BWD=fused."""
    ga, gb = _default_and_pool(oracle_params, "attack_grad")
    assert torch.equal(ga, gb), float((ga - gb).abs().max())
