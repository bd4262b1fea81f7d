"""Throughput of the weight-gradient pass (dp_eot_backward_params) against the forward, the input-only backward and
PyTorch eager on the same GPU, at 224 px, chunk 128, library algorithms by heuristic (autotune off).

    python tools/param_grad_bench.py [--precisions tf32,bf16] [--iters 5] [--warmup 2] [--out results.json]

Shapes: B=128 x S=1 (a fine-tuning batch, two cutout rectangles per image) and B=1 x S=128 (EOT).  Rows (samples/s):
fwd, fwd + input backward, fwd + input + weight backward, fwd + weight-only backward (no input gradient), and torch
eager (the oracle on CUDA: cuDNN with TF32 convolutions, or bf16 autocast; weights and input gradients).  Then the
engine's per-category profile of one fwd + input + weight backward call."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dorpatch_b200.engine import Engine  # noqa: E402
from oracle import resnetv2 as OR  # noqa: E402

H = 224


def cutout_rects(B, S, rs):
    r = np.zeros((B, S, 4, 4), np.int16)
    for b in range(B):
        for s in range(S):
            for k in range(2):
                a, c = rs.randint(0, H - 128, 2)
                r[b, s, k] = (a, a + 128, c, c + 128)
    return r


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="tf32,bf16")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    params = OR.random_init(seed=0, affine_jitter=0.1)
    names = list(params)
    rows = []
    for prec in a.precisions.split(","):
        eng = Engine(img=H, precision=prec, chunk=128, max_images=128, autotune=False)
        eng.load_state_dict(params)
        grads = [torch.zeros(params[k].shape, device="cuda") for k in names]
        for B, S in ((128, 1), (1, 128)):
            rs = np.random.RandomState(0)
            img = torch.rand(B, 3, H, H, device="cuda")
            rects = cutout_rects(B, S, rs)
            dl = (torch.rand(B * S, 1000, device="cuda") - 0.5) / (B * S)
            N = B * S
            res = {}
            res["fwd"] = timed(lambda: eng.eot_forward(img, S, rects), a.iters, a.warmup)
            res["fwd+dx"] = timed(lambda: (eng.eot_forward(img, S, rects), eng.eot_backward(dl)), a.iters, a.warmup)
            res["fwd+dx+dW"] = timed(lambda: (eng.eot_forward(img, S, rects),
                                              eng.eot_backward_params(dl, names, grads, grad_img=True)), a.iters, a.warmup)
            res["fwd+dW"] = timed(lambda: (eng.eot_forward(img, S, rects),
                                           eng.eot_backward_params(dl, names, grads, grad_img=False)), a.iters, a.warmup)
            on = OR.OracleNet({k: v.cuda() for k, v in params.items()}, weights_require_grad=True).cuda()
            keep = torch.ones(B, S, 1, H, H, dtype=torch.bool, device="cuda")
            for b in range(B):
                for s in range(S):
                    for k in range(2):
                        r0, r1, c0, c1 = [int(v) for v in rects[b, s, k]]
                        keep[b, s, 0, r0:r1, c0:c1] = False
            torch.backends.cudnn.allow_tf32 = True
            torch.backends.cuda.matmul.allow_tf32 = prec == "tf32"

            def eager():
                x = img.clone().requires_grad_(True)
                xs = torch.where(keep, x[:, None], torch.full_like(x[:, None], 0.5)).reshape(N, 3, H, H)
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=prec == "bf16"):
                    out = on(xs)
                (out.float() * dl).sum().backward()
                on.zero_grad(set_to_none=True)
            res["torch_eager"] = timed(eager, a.iters, a.warmup)
            del on
            torch.cuda.empty_cache()
            eng.profile(True, reset=True)
            eng.eot_forward(img, S, rects)
            eng.eot_backward_params(dl, names, grads, grad_img=True)
            prof = eng.profile_read()
            eng.profile(False)
            row = dict(precision=prec, B=B, S=S, samples_per_s={k: round(N / (ms * 1e-3), 1) for k, ms in res.items()},
                       ms={k: round(ms, 3) for k, ms in res.items()},
                       profile={k: dict(ms=round(v["ms"], 3), count=v["count"],
                                        gbs=round(v["bytes"] / (v["ms"] * 1e-3) / 1e9, 1) if v["ms"] > 0 else 0.0,
                                        tflops=round(v["flops"] / (v["ms"] * 1e-3) / 1e12, 2) if v["ms"] > 0 else 0.0)
                                for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])})
            print(json.dumps(row), flush=True)
            rows.append(row)
        eng.close()
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
