"""Cost of the stage-0 step at several basic_units on one GPU, one JSON line.

    python tools/basic_unit_bench.py [--precisions tf32,bf16] [--units 1,7,14,28] [--steps 10]

On a random-init ResNetV2-50x1-BiT at 224 px, per precision, for B=1 x S=128 and c3 (B=64 x S=32), per unit u:
  ms_per_step       steady-state stage-0 step (dp_attack_grad + dp_attack_update, random mask, EOT samples from the
                    one-patch dropout-2 universe), CUDA graphs on, profiler off
  maskreg_ms        per step, the density / group-lasso kernel (engine profiler category `maskreg`, a separate run)
  update_ms         per step, the K3 sign-step kernel (`update_k3`), which reads the group sums of squares at u
  maskreg_share     maskreg_ms / ms_per_step
Library algorithms come from the heuristics (no timing trials), as in bench.py.  Every timed shape is warmed up first.
The GPU's name and power limit are read in the same process.
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
from dorpatch_b200.engine import Engine               # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2           # noqa: E402
from tools.pc_bench import gpu_info                   # noqa: E402

IMG = 224
SHAPES = {"B1xS128": (1, 128), "c3_B64xS32": (64, 32)}


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def unit_leg(eng, B, S, u, steps):
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    pattern = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    mask = torch.rand(B, 1, IMG, IMG, generator=g).cuda()
    G = torch.zeros_like(x)
    y = (eng.predict(x).astype(np.int64) + 1) % 1000
    table = PM.universe(IMG, 2)
    rng = np.random.RandomState(0)
    rects = [PM.gather(table, np.stack([rng.choice(len(table), S, replace=False) for _ in range(B)]))
             for _ in range(steps)]
    lr, st, cg = np.full(B, 1e-4, np.float32), [1e-3] * B, [1e-5] * B

    def step(i):
        eng.attack_grad(x, mask, pattern, rects[i % steps], y, [True] * B, 0.1, 4.0, 0, G, S_total=S, basic_unit=u)
        eng.attack_update(x, mask, pattern, G, lr, st, cg, 1e-3, 0)

    timed(step, 5)
    s = timed(step, steps)
    eng.profile(True, reset=True)
    n_prof = min(steps, 5)
    timed(step, n_prof)
    prof = eng.profile_read()
    eng.profile(False)
    mr, up = prof["maskreg"]["ms"] / n_prof, prof["update_k3"]["ms"] / n_prof
    return {"ms_per_step": s * 1e3, "samples_per_s": B * S / s, "maskreg_ms": mr, "update_ms": up,
            "maskreg_share": mr / (s * 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="tf32,bf16")
    ap.add_argument("--units", default="1,7,14,28")
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/basic_unit_bench.py needs a CUDA device (H100)")
    torch.cuda.set_device(0)
    sd = ResNetV2(seed=0).state_dict()
    units = [int(u) for u in args.units.split(",")]
    out = {"tool": "basic_unit_bench", "img": IMG, "model": "ResNetV2-50x1-BiT random-init (seed 0)", "gpu": gpu_info(),
           "legs": {}}
    for prec in args.precisions.split(","):
        leg = {}
        for shape, (B, S) in SHAPES.items():
            eng = Engine(img=IMG, precision=prec, chunk=128, max_images=B, autotune=False)
            eng.load_state_dict(sd)
            leg[shape] = {"u%d" % u: unit_leg(eng, B, S, u, args.steps) for u in units}
            eng.close()
        out["legs"][prec] = leg
    print(json.dumps(out))


if __name__ == "__main__":
    main()
