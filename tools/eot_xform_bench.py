"""Cost of affine / colour EOT through the differentiable classifier, one JSON line.

    python tools/eot_xform_bench.py [--precisions tf32,bf16] [--steps 5] [--warmup 2]

On a random-init ResNetV2-50x1-BiT at 224 px, engine chunk 128, per precision, for B=1 x S=128 and c3 (B=64 x S=32),
every step with fresh transforms (eot.sample, affine 0.5, colour 0.5) and fresh two-rectangle occlusions:
  eot_xform    eot_logits(model, adv, rects, S, xforms=...) + cross-entropy backward: dp_eot_forward_xform +
               dp_eot_backward, the warp and its adjoint in the engine (expand_affine / reduce_affine)
  attack_grad  dp_attack_grad (stage 1) with the same transforms: the fixed CW loss generate optimises
  torch_warp   what a user had to write before: F.affine_grid + F.grid_sample + the colour clamp on B*S fp32 images in
               torch, then eot_logits with S = 1 on an engine with max_images = B*S, cross-entropy backward through both
Each leg reports ms per step and EOT samples/s, the two eot_logits legs also their engine's device memory (MB);
`vs_torch_warp` is eot_xform's rate over torch_warp's, and `logit_max_abs_diff` compares eot_xform's logits with
torch_warp's on the first step's inputs.  Library algorithms come from the heuristics (no timing trials), as in bench.py.
Every timed shape is warmed up first.  The GPU's name and power limit are read in the same process.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dorpatch_b200 import eot as PE                   # noqa: E402
from dorpatch_b200 import masks as PM                 # noqa: E402
from dorpatch_b200.engine import Engine               # noqa: E402
from dorpatch_b200.ops import eot_logits              # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2           # noqa: E402
from tools.pc_bench import gpu_info                   # noqa: E402

IMG, CHUNK = 224, 128
SHAPES = {"B1xS128": (1, 128), "c3_B64xS32": (64, 32)}


def timed(fn, n, start):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        fn(start + i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def torch_warp(adv, xf):
    """oracle/eot.py's transform on the device: [B,3,H,W], [B,S,8] -> [B*S,3,H,W]."""
    B, _, H, W = adv.shape
    S = xf.shape[1]
    theta = xf[..., :6].reshape(B * S, 2, 3)
    grid = F.affine_grid(theta, (B * S, 3, H, W), align_corners=False)
    src = adv[:, None].expand(B, S, 3, H, W).reshape(B * S, 3, H, W)
    warped = F.grid_sample(src, grid, mode="bilinear", padding_mode="border", align_corners=False)
    c, b = xf[..., 6].reshape(B * S, 1, 1, 1), xf[..., 7].reshape(B * S, 1, 1, 1)
    return torch.clamp(c * (warped - 0.5) + 0.5 + b, 0.0, 1.0)


def legs(prec, sd, B, S, steps, warmup):
    n_draw = steps + warmup
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    pattern = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    mask = torch.rand(B, 1, IMG, IMG, generator=g).cuda()
    table = PM.universe(IMG, 2)
    rng = np.random.RandomState(0)
    rects = [PM.gather(table, rng.randint(0, len(table), (B, S))) for _ in range(n_draw)]
    xfs = [PE.sample(rng, B, S, 0.5, 0.5) for _ in range(n_draw)]
    xfs_dev = [torch.from_numpy(xf).cuda() for xf in xfs]

    eng = Engine(img=IMG, precision=prec, chunk=CHUNK, max_images=B, autotune=False)
    eng.load_state_dict(sd)
    net = ResNetV2(seed=0)
    net.adopt_engine(eng)
    G = torch.zeros_like(x)
    y = (eng.predict(x).astype(np.int64) + 1) % 1000
    yy = torch.from_numpy(np.repeat(y, S)).cuda()
    adv, _, _ = eng.paste(x, mask, pattern, 4.0)
    out = {}

    def eot_xform(i):
        a = adv.detach().requires_grad_(True)
        F.cross_entropy(eot_logits(net, a, rects[i], S, xforms=xfs[i]), yy).backward()

    def attack(i):
        eng.attack_grad(x, mask, pattern, rects[i], y, [True] * B, 0.1, 4.0, 1, G, S_total=S, xforms=xfs[i])

    for name, fn in (("eot_xform", eot_xform), ("attack_grad", attack)):
        timed(fn, warmup, 0)
        s = timed(fn, steps, warmup)
        out[name] = {"ms_per_step": s * 1e3, "samples_per_s": B * S / s}
    with torch.no_grad():
        l_native = eng.eot_forward(adv, S, rects[0], xforms=xfs[0]).cpu()
    out["eot_xform"]["engine_mb"] = eng.device_bytes / 2 ** 20
    eng.close()
    torch.cuda.empty_cache()

    eng_w = Engine(img=IMG, precision=prec, chunk=CHUNK, max_images=B * S, autotune=False)
    eng_w.load_state_dict(sd)
    net_w = ResNetV2(seed=0)
    net_w.adopt_engine(eng_w)

    def warp(i):
        a = adv.detach().requires_grad_(True)
        w = torch_warp(a, xfs_dev[i])
        F.cross_entropy(eot_logits(net_w, w, rects[i].reshape(B * S, 1, 4, 4), 1), yy).backward()

    timed(warp, warmup, 0)
    s = timed(warp, steps, warmup)
    out["torch_warp"] = {"ms_per_step": s * 1e3, "samples_per_s": B * S / s, "engine_mb": eng_w.device_bytes / 2 ** 20}
    with torch.no_grad():
        l_warp = eng_w.eot_forward(torch_warp(adv, xfs_dev[0]).contiguous(), 1, rects[0].reshape(B * S, 1, 4, 4)).cpu()
    eng_w.close()
    torch.cuda.empty_cache()
    out["vs_torch_warp"] = out["eot_xform"]["samples_per_s"] / out["torch_warp"]["samples_per_s"]
    out["vs_attack_grad"] = out["eot_xform"]["samples_per_s"] / out["attack_grad"]["samples_per_s"]
    out["logit_max_abs_diff"] = float((l_native - l_warp).abs().max())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="tf32,bf16")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/eot_xform_bench.py needs a CUDA device (H100)")
    torch.cuda.set_device(0)
    sd = ResNetV2(seed=0).state_dict()
    out = {"tool": "eot_xform_bench", "img": IMG, "chunk": CHUNK, "model": "ResNetV2-50x1-BiT random-init (seed 0)",
           "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(), "legs": {}}
    for prec in args.precisions.split(","):
        out["legs"][prec] = {shape: legs(prec, sd, B, S, args.steps, args.warmup) for shape, (B, S) in SHAPES.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
