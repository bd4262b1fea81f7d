"""Cost of generating against the two-patch PatchCleanser window on one GPU, one JSON line.

    python tools/two_patch_gen_bench.py [--precisions tf32,bf16] [--steps 10]

On a random-init ResNetV2-50x1-BiT at 224 px, per precision:
  step      steady-state stage-1 step (dp_attack_grad + dp_attack_update, the EOT samples gathered from the universe) for
            B=1 x S=128 and c3 (B=64 x S=32), samples drawn from the two-patch dropout-2 universe (90 720 masks, 3
            rectangles each) against the one-patch universe (2 520 masks, 2 rectangles); ms per step and samples/s.
  scan      one universe scan of one image: dp_predict over the 31 080 distinct occlusions (what generate runs) against
            all 90 720 masks, and a plain dp_predict over the 2 520-mask one-patch universe as the rate yardstick.
and once, without the network (random losses, 60 % of the samples succeed):
  host      host milliseconds per step at B=64 x S=32 in the i >= 1000 regime over the two-patch universe (half of each
            image's samples drawn from its failed set, initially 9 072 masks): failed sets as device bitmaps
            (dp_failed_set_update + dp_failed_set_read, as generate runs them) against host lists (DORPATCH_FAILED=host),
            and the numpy draw alone (the rng.choice over 90 720 indices per image that must stay on the host).
Library algorithms come from the heuristics (no timing trials), as in bench.py.  Every timed shape is warmed up first.  The GPU's name and power limit are read in the same process.
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


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def step_leg(eng, table, B, S, steps):
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    pattern = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    mask = DorPatch().patch_selection(torch.rand(B, 1, IMG, IMG, generator=g).cuda(), 0.12)
    G = torch.zeros_like(x)
    y = (eng.predict(x).astype(np.int64) + 1) % 1000
    rng = np.random.RandomState(0)
    rects = [PM.gather(table, np.stack([rng.choice(len(table), S, replace=False) for _ in range(B)]))
             for _ in range(steps)]
    lr, st, cg = np.full(B, 0.01, np.float32), [1e-3] * B, [1e-5] * B

    def step(i):
        eng.attack_grad(x, mask, pattern, rects[i % steps], y, [True] * B, 0.1, 4.0, 1, G, S_total=S)
        eng.attack_update(x, mask, pattern, G, lr, st, cg, 1e-3, 1)

    timed(step, 5)
    s = timed(step, steps)
    return {"ms_per_step": s * 1e3, "samples_per_s": B * S / s}


def scan_leg(eng, reps=2):
    img = torch.rand(1, 3, IMG, IMG, generator=torch.Generator().manual_seed(7)).cuda()
    two = PM.universe(IMG, 2, 2)
    distinct, _ = PM.distinct_occlusions(two, len(PM.DROPOUT_SIZES))
    sets = {"distinct_31080": PM.gather(distinct, np.arange(len(distinct))), "full_90720": PM.gather(two, np.arange(len(two))),
            "one_patch_2520": PM.gather(PM.universe(IMG, 2), np.arange(2520))}
    out = {}
    eng.predict(img, 2520, sets["one_patch_2520"])                     # warm-up: every dp_predict chunk shape
    for name, r in sets.items():
        s = min(timed(lambda i: eng.predict(img, len(r), r), 1) for _ in range(reps))
        out[name] = {"s": s, "forwards_per_s": len(r) / s}
    for name in ("distinct_31080", "full_90720"):
        out[name]["rate_vs_dp_predict_2520"] = out[name]["forwards_per_s"] / out["one_patch_2520"]["forwards_per_s"]
    out["distinct_vs_full_speedup"] = out["full_90720"]["s"] / out["distinct_31080"]["s"]
    return out


def host_leg(eng, B=64, S=32, steps=30):
    n_mask = len(PM.universe(IMG, 2, 2))
    out = {}
    for mode in ("device", "host"):
        rng = np.random.RandomState(0)
        states = [_ImageState(0.01, 1e-3, 3, False, np.random.RandomState(10 + b)) for b in range(B)]
        if mode == "device":
            eng.failed_reset(n_mask)
            for b, s in enumerate(states):
                s.dev = (eng, b)
        for s in states:
            s.set_failed(sorted(rng.choice(n_mask, n_mask // 10, replace=False).tolist()))
        losses = [(rng.rand(B, S) < 0.6).astype(np.float32) * 0.5 for _ in range(steps)]
        t_draw = t_all = 0.0
        for i in range(1000, 1000 + steps):
            t0 = time.perf_counter()
            drawn = [s.sample(i, n_mask, S) for s in states]
            t1 = time.perf_counter()
            idx, nff = np.stack([d[0] for d in drawn]), [d[1] for d in drawn]
            loss = losses[i - 1000]
            counts = eng.failed_update(idx, nff, [True] * B, loss=loss) if mode == "device" else [None] * B
            for b, s in enumerate(states):
                s.bookkeeping(1, i, loss[b], idx[b], nff[b], 1.0, n_failed=counts[b])
            t2 = time.perf_counter()
            t_draw += t1 - t0
            t_all += t2 - t0
        out[mode] = {"ms_per_step": t_all / steps * 1e3, "ms_sampling": t_draw / steps * 1e3,
                     "mean_failed_set": float(np.mean([s.n_failed for s in states]))}
    t0 = time.perf_counter()
    rs = np.random.RandomState(0)
    for _ in range(steps):
        for _ in range(B):
            rs.choice(np.arange(n_mask), S // 2, replace=False)
    out["numpy_universe_draw_ms_per_step"] = (time.perf_counter() - t0) / steps * 1e3
    out["note"] = "B=%d x S=%d, i >= 1000, %d steps; sampling = the numpy draws (+ dp_failed_set_read on device)" % (B, S, steps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="tf32,bf16")
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/two_patch_gen_bench.py needs a CUDA device (H100)")
    torch.cuda.set_device(0)
    sd = ResNetV2(seed=0).state_dict()
    tables = {"two_patch_90720": PM.universe(IMG, 2, 2), "one_patch_2520": PM.universe(IMG, 2)}
    out = {"tool": "two_patch_gen_bench", "img": IMG, "model": "ResNetV2-50x1-BiT random-init (seed 0)", "gpu": gpu_info(),
           "legs": {}}
    for prec in args.precisions.split(","):
        leg = {}
        for shape, (B, S) in SHAPES.items():
            eng = Engine(img=IMG, precision=prec, chunk=128, max_images=B, autotune=False)
            eng.load_state_dict(sd)
            leg[shape] = {name: step_leg(eng, t, B, S, args.steps) for name, t in tables.items()}
            if B == 1:
                leg["scan"] = scan_leg(eng)
            else:
                if "host" not in out:
                    out["host"] = host_leg(eng)
            eng.close()
        out["legs"][prec] = leg
    print(json.dumps(out))


if __name__ == "__main__":
    main()
