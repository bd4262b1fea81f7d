"""Workload for compute-sanitizer (tools/sanitize.sh): every hand-written kernel family once, at sizes the tools finish in
about a minute -- K1 (bulk-copy tiles + mbarriers), the cluster GroupNorm kernels (TMA slab, DSMEM reduce, split cluster
barriers) through dp_debug_gn at cluster-1 / multi-CTA shapes, the bf16 stem kernels, one whole stage-0 and stage-1 attack
step (paste, K1, net forward/backward, CW, fused stem-dgrad + reduce, regularisers, sign step), dp_predict, one
dp_eot_forward_xform + dp_eot_backward (affine expansion and its atomic adjoint), the failed-set bitmaps.  usage: python tools/sanitize_run.py [bf16|fp32|tf32] [img]"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dorpatch_b200 import _lib, masks as PM                       # noqa: E402
from dorpatch_b200.engine import Engine                           # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2                       # noqa: E402


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def main():
    prec = sys.argv[1] if len(sys.argv) > 1 else "bf16"
    img = int(sys.argv[2]) if len(sys.argv) > 2 else 112
    light = len(sys.argv) > 3 and sys.argv[3] == "light"     # racecheck is ~100x slower: skip the whole-network steps
    torch.cuda.set_device(0)
    dev = "cuda:0"
    B, S = 2, 3
    eng = Engine(img=img, precision=prec, chunk=4, max_images=B, device=0, autotune=False)
    eng.load_state_dict(ResNetV2(seed=0).state_dict())
    g = torch.Generator().manual_seed(1)
    x, m, p = (torch.rand(B, 3, img, img, generator=g).to(dev), torch.rand(B, 1, img, img, generator=g).to(dev),
               torch.rand(B, 3, img, img, generator=g).to(dev))
    table = PM.universe(img, 2)
    idx = np.random.RandomState(0).randint(0, table.shape[0], (B, S))
    rects = PM.gather(table, idx)
    y = eng.predict(x).astype(np.int64) if not light else np.array([1, 2])
    G = torch.zeros_like(x)
    for stage in (() if light else (0, 1)):
        r = eng.attack_grad(x, m, p, rects, y, [False] * B, 0.1, 4.0, stage, G)
        eng.attack_update(x, m, p, G, np.full(B, 0.01, np.float32), [1e-3] * B, [1e-5] * B, 1e-3, stage)
        assert np.isfinite(r["loss_adv"]).all()
    if not light:
        eng.predict(x, S, rects)
        # the differentiable classifier under affine / colour EOT: expand_affine, unfused stem dgrad, reduce_affine
        # (two chunks, the first recomputed in the backward)
        from dorpatch_b200 import eot as PE
        logits = eng.eot_forward(x, S, rects, xforms=PE.sample(np.random.RandomState(1), B, S, 0.5, 0.5))
        eng.eot_backward(torch.randn_like(logits))
        # the weight-gradient pass over every parameter (two chunks, the first recomputed), with and without the input
        # gradient: recomputed GroupNorm inputs, GroupNorm affine partials, stem / 1x1 / 3x3 / fc wgrad, WS adjoint
        from dorpatch_b200.resnetv2 import param_shapes
        shapes = param_shapes(1000)
        names = list(shapes)
        grads = [torch.zeros(shapes[k], device=dev) for k in names]
        logits = eng.eot_forward(x, S, rects)
        eng.eot_backward_params(torch.randn_like(logits), names, grads, grad_img=True)
        eng.eot_backward_params(torch.randn_like(logits), names, grads, grad_img=False, accumulate=True)
    eng.expand(x, S, rects)
    eng.paste(x, m, p, 4.0)
    # the in-step K1 variant (paste fused in), both store paths
    rd = torch.from_numpy(np.ascontiguousarray(rects.reshape(B * S, 4, 4), np.int16)).to(dev)
    out = torch.empty((B * S, img, img, eng.c_pad), dtype=torch.bfloat16 if eng.elem_bytes == 2 else torch.float32, device=dev)
    for mode in (0, 1):
        eng.lib.dp_debug_k1_tuning(0, 0, mode)
        _lib.check(eng.lib.dp_expand_step_dev(eng.handle, ptr(x), ptr(m), ptr(p), B, S, ptr(rd), 0, B * S, ptr(out), eng._stream()))
    eng.lib.dp_debug_k1_tuning(0, 0, 0)
    eng.window_sum(m, 7)
    eng.failed_write(0, [1, 5, 9])
    eng.failed_update(idx, [0] * B, [True] * B, loss=np.random.rand(B, S).astype(np.float32))
    eng.failed_read(0)
    dt = torch.bfloat16 if eng.elem_bytes == 2 else torch.float32
    for P, Cc in ((784, 128), (3136, 64), (196, 1024), (49, 2048)):
        N = 2
        xd = torch.randn(N, P, Cc, device=dev).to(dt)
        dyd = torch.randn(N, P, Cc, device=dev).to(dt)
        add = torch.randn(N, P, Cc, device=dev).to(dt)
        gd, bd = torch.rand(Cc, device=dev) + 0.5, torch.randn(Cc, device=dev) * 0.1
        yv, dx = torch.empty_like(xd), torch.empty_like(xd)
        stats = torch.empty(N, 32, 2, device=dev)
        _lib.check(eng.lib.dp_debug_gn(eng.handle, ptr(xd), ptr(dyd), ptr(add), ptr(gd), ptr(bd), 1, ptr(yv), ptr(dx), ptr(stats), N, P, Cc,
                                       eng._stream()))
    torch.cuda.synchronize()
    eng.close()
    print("sanitize_run ok", prec, img, "light" if light else "full")


if __name__ == "__main__":
    main()
