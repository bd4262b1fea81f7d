"""Cost of the differentiable classifier (dp_eot_forward + dp_eot_backward) against dp_attack_grad, one JSON line.

    python tools/autograd_bench.py [--precisions tf32,bf16] [--steps 10]

On a random-init ResNetV2-50x1-BiT at 224 px, engine chunk 128, per precision, for B=1 x S=128 and c3 (B=64 x S=32):
  attack_grad       dp_attack_grad (stage 1: no mask regularisers) with CUDA graphs on, as generate runs it
  eot               eot_forward + a CW gradient formed in torch + eot_backward, what a user loop over
                    ops.eot_logits costs; chunks beyond the two the lanes hold are recomputed in the backward
  eot_ratio         eot samples/s over attack_grad samples/s
  recomputed_chunks chunks the backward runs the forward for again (all chunks minus the two resident ones)
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

IMG, CHUNK = 224, 128
SHAPES = {"B1xS128": (1, 128), "c3_B64xS32": (64, 32)}


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def cw_dlogits(logits, y, w, confidence=0.1):
    """Targeted CW gradient (attack.py:16-23) of w * sum of the losses."""
    n = torch.arange(logits.shape[0], device=logits.device)
    real = logits[n, y]
    oi = logits.scatter(1, y[:, None], float("-inf")).argmax(1)
    live = (confidence + logits[n, oi] - real) >= 0
    d = torch.zeros_like(logits)
    d[n, y] = torch.where(live, -w, 0.0)
    d[n, oi] = torch.where(live, w, 0.0)
    return d


def legs(eng, B, S, steps):
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    pattern = torch.rand(B, 3, IMG, IMG, generator=g).cuda()
    mask = torch.rand(B, 1, IMG, IMG, generator=g).cuda()
    G = torch.zeros_like(x)
    y = (eng.predict(x).astype(np.int64) + 1) % 1000
    yy = torch.from_numpy(np.repeat(y, S)).cuda()
    table = PM.universe(IMG, 2)
    rng = np.random.RandomState(0)
    rects = [PM.gather(table, np.stack([rng.choice(len(table), S, replace=False) for _ in range(B)]))
             for _ in range(steps)]
    adv, _, _ = eng.paste(x, mask, pattern, 4.0)

    def attack(i):
        eng.attack_grad(x, mask, pattern, rects[i % steps], y, [True] * B, 0.1, 4.0, 1, G, S_total=S)

    def eot(i):
        logits = eng.eot_forward(adv, S, rects[i % steps])
        eng.eot_backward(cw_dlogits(logits, yy, 1.0 / S), out=G)

    out = {}
    for name, fn in (("attack_grad", attack), ("eot", eot)):
        timed(fn, 3)
        s = timed(fn, steps)
        out[name] = {"ms_per_step": s * 1e3, "samples_per_s": B * S / s}
    out["eot_ratio"] = out["eot"]["samples_per_s"] / out["attack_grad"]["samples_per_s"]
    out["recomputed_chunks"] = max(0, -(-B * S // CHUNK) - 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="tf32,bf16")
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/autograd_bench.py needs a CUDA device (H100)")
    torch.cuda.set_device(0)
    sd = ResNetV2(seed=0).state_dict()
    out = {"tool": "autograd_bench", "img": IMG, "chunk": CHUNK, "model": "ResNetV2-50x1-BiT random-init (seed 0)",
           "gpu": gpu_info(), "legs": {}}
    for prec in args.precisions.split(","):
        leg = {}
        for shape, (B, S) in SHAPES.items():
            eng = Engine(img=IMG, precision=prec, chunk=CHUNK, max_images=B, autotune=False)
            eng.load_state_dict(sd)
            leg[shape] = legs(eng, B, S, args.steps)
            eng.close()
        out["legs"][prec] = leg
    print(json.dumps(out))


if __name__ == "__main__":
    main()
