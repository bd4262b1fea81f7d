"""Host sampler against device sampler in generate()'s step at i >= 1000, one JSON line.

    python tools/device_sampler_bench.py [--precisions tf32,bf16] [--steps 8]

On a random-init ResNetV2-50x1-BiT at 224 px, stage 1, per precision, shape (B=1 x S=128, c3 = B=64 x S=32) and universe
(two-patch dropout-2: 90 720 masks; one-patch dropout-2: 2 520), each image's failed set initially a random tenth of the
universe, so half of every image's samples come from it.  One step is what generate() runs:
  host    per image _ImageState.sample (dp_failed_set_read + the numpy draws) and masks.gather, dp_attack_grad,
          dp_failed_set_update, the bookkeeping, dp_attack_update;
  device  dp_eot_draw, dp_attack_grad_drawn, dp_failed_set_update_drawn, the bookkeeping, dp_attack_update.
Reported per step: wall ms (host clock; every step ends in a device synchronise), host ms (the sampling / draw call,
the failed-set update call and the bookkeeping: the part of the step the GPU waits for, since the gradient call
synchronises) and the GPU-side ms (the two engine calls).  Then the draw kernel's time from the engine profiler, in a
run of its own.  Library algorithms come from the heuristics, as in bench.py.  The GPU's name and power limit are read
in the same process.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dorpatch_b200 import masks as PM                 # noqa: E402
from dorpatch_b200.attack import DorPatch, _ImageState  # noqa: E402
from dorpatch_b200.engine import Engine               # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2           # noqa: E402
from tools.pc_bench import gpu_info                   # noqa: E402

IMG = 224
SHAPES = {"B1xS128": (1, 128), "c3_B64xS32": (64, 32)}


def run_leg(eng, table, B, S, sampler, steps, warmup=3):
    n_mask = len(table)
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    pattern = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    mask = DorPatch().patch_selection(torch.rand(B, 1, IMG, IMG, generator=g).cuda(), 0.12)
    G = torch.zeros_like(x)
    y = (eng.predict(x).astype(np.int64) + 1) % 1000
    rng = np.random.RandomState(0)
    st = [_ImageState(0.01, 1e-3, int(y[b]), True, np.random.RandomState(10 + b)) for b in range(B)]
    eng.failed_reset(n_mask)
    eng.eot_universe(table)
    for b, s in enumerate(st):
        s.dev = (eng, b)
        s.set_failed(sorted(rng.choice(n_mask, n_mask // 10, replace=False).tolist()))
    seeds = list(range(100, 100 + B))
    t_wall = t_host = t_gpu = 0.0
    for k in range(warmup + steps):
        i = 1000 + k
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if sampler == "host":
            drawn = [s.sample(i, n_mask, S) for s in st]
            idx, nff = np.stack([d[0] for d in drawn]), [d[1] for d in drawn]
            rects = PM.gather(table, idx)
        else:
            eng.eot_draw(seeds, 1, i, [True] * B, S)
            rects = None
        t1 = time.perf_counter()
        r = eng.attack_grad(x, mask, pattern, rects, y, [True] * B, 0.1, 4.0, 1, G, S_total=S, S=S)
        t2 = time.perf_counter()
        if sampler == "host":
            counts = eng.failed_update(idx, nff, [True] * B)
        else:
            counts = eng.failed_update_drawn(B, S, [True] * B)
        lr = np.zeros(B, np.float32)
        for b, s in enumerate(st):
            s.bookkeeping(1, i, r["loss_adv"][b], None, None, r["loss_struc"][b], n_failed=counts[b])
            lr[b] = s.lr
        t3 = time.perf_counter()
        eng.attack_update(x, mask, pattern, G, lr, [s.structured for s in st], [s.coeff_group_lasso for s in st],
                          1e-3, 1)
        t4 = time.perf_counter()
        if k >= warmup:
            t_wall += t4 - t0
            t_host += (t1 - t0) + (t3 - t2)
            t_gpu += (t2 - t1) + (t4 - t3)
    return {"ms_per_step": t_wall / steps * 1e3, "host_ms": t_host / steps * 1e3, "gpu_calls_ms": t_gpu / steps * 1e3,
            "mean_failed_set": float(np.mean([s.n_failed for s in st]))}


def draw_kernel_ms(eng, table, B, S, reps=20):
    eng.failed_reset(len(table))
    eng.eot_universe(table)
    rng = np.random.RandomState(1)
    for b in range(B):
        eng.failed_write(b, rng.choice(len(table), len(table) // 10, replace=False))
    eng.eot_draw(list(range(B)), 1, 1000, [True] * B, S)
    eng.profile(True, reset=True)
    for k in range(reps):
        eng.eot_draw(list(range(B)), 1, 1001 + k, [True] * B, S)
    torch.cuda.synchronize()
    p = eng.profile_read().get("eot_draw", {"ms": float("nan"), "count": 1})
    eng.profile(False)
    return p["ms"] / max(p["count"], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="tf32,bf16")
    ap.add_argument("--steps", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/device_sampler_bench.py needs a CUDA device (H100)")
    torch.cuda.set_device(0)
    sd = ResNetV2(seed=0).state_dict()
    tables = {"two_patch_90720": PM.universe(IMG, 2, 2), "one_patch_2520": PM.universe(IMG, 2)}
    out = {"tool": "device_sampler_bench", "img": IMG, "model": "ResNetV2-50x1-BiT random-init (seed 0)", "gpu": gpu_info(),
           "legs": {}, "draw_kernel_ms": {}}
    for prec in args.precisions.split(","):
        leg = {}
        for shape, (B, S) in SHAPES.items():
            eng = Engine(img=IMG, precision=prec, chunk=128, max_images=B, autotune=False)
            eng.load_state_dict(sd)
            for name, t in tables.items():
                leg["%s/%s" % (shape, name)] = {smp: run_leg(eng, t, B, S, smp, args.steps) for smp in ("host", "device")}
                if prec == args.precisions.split(",")[0]:
                    out["draw_kernel_ms"]["%s/%s" % (shape, name)] = draw_kernel_ms(eng, t, B, S)
            eng.close()
        out["legs"][prec] = leg
    print(json.dumps(out))


if __name__ == "__main__":
    main()
