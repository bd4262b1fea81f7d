"""Mask bank against rectangle tables on the same occlusions, on one GPU.  Prints one JSON object.

    python tools/mask_bank_bench.py [--img 224] [--reps 5]

Workload: `predict` of one image over the one-patch dropout-2 universe (2 520 masks) as the rectangle table and as a
mask bank of the same occlusions, on a bf16 engine (tight c3 input) and a tf32 engine (c4), chunk 64.

- K1 kernel time at the launch size `predict` uses (one launch per 64-sample chunk): the engine profiler's
  `expand_k1` / `expand_k1_bank` categories (CUDA events around each launch) over `reps` whole `predict` calls
  (40 launches each) after a warm-up call, and the share of the HBM peak (3.35 TB/s): physical bytes = the samples
  written (H*W*Cp*elem), the image planes read once per launch, and for the bank one mask's words plus the index pair
  per sample.  The profiler runs the chunks on one lane; the host staging of rectangles / indices lies outside the
  timed launches.
- `predict` over the universe, profiler off, in forwards/s (`reps` calls after a warm-up, host clock around each call,
  which ends in a device synchronisation).
- `eot_forward` + `eot_backward` at B x S = 1 x 128 and 64 x 32 (bf16), bank and rectangles, in ms per pair.
- dp_engine_device_bytes of a fresh engine, after rectangle calls and after bank calls; the bank's own size.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dorpatch_b200 import masks as PM  # noqa: E402
from dorpatch_b200.engine import Engine  # noqa: E402
from oracle import resnetv2 as OR  # noqa: E402

DEV = "cuda:0"
HBM = 3.35e12


def _host_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / reps


def _kernel_ms(e, cat, fn, reps):
    """Mean time of one launch of profiler category `cat` over `reps` calls of fn (after one warm-up call)."""
    fn()
    torch.cuda.synchronize()
    e.profile(True, reset=True)
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    r = e.profile_read()[cat]
    e.profile(False, reset=True)
    return r["ms"] / r["count"], r["count"] // reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--img", type=int, default=224)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    H = args.img
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    params = OR.random_init(seed=0)
    table = PM.universe(H, 2)                                    # [2520,2,4]
    n = len(table)
    rects = PM.gather(table, np.arange(n))
    bank = PM.pack_bank(PM.to_bool(table, H), device=DEV)
    idx = np.arange(n)
    img = torch.rand(1, 3, H, H, generator=torch.Generator().manual_seed(0)).to(DEV)
    out = {"card": card, "img": H, "bank_bytes": bank.numel() * 4, "masks": n}
    for prec in ("bf16", "tf32"):
        e = Engine(img=H, precision=prec, chunk=64, max_images=64, autotune=False)
        e.load_state_dict(params)
        dev0 = e.device_bytes
        pr = lambda: e.predict(img, n, rects)                   # noqa: E731
        pb = lambda: e.predict(img, n, bank=bank, idx=idx)      # noqa: E731
        ms_pr = _host_ms(pr, args.reps)
        dev1 = e.device_bytes
        ms_pb = _host_ms(pb, args.reps)
        dev2 = e.device_bytes
        k_r, launches = _kernel_ms(e, "expand_k1", pr, args.reps)
        k_b, _ = _kernel_ms(e, "expand_k1_bank", pb, args.reps)
        per = n / launches                                       # samples per launch
        written = per * H * H * e.c_pad * e.elem_bytes + 3 * H * H * 4
        bank_read = per * (H * PM.bank_words(H) * 4 + 8)
        out["k1_%s_c%d" % (prec, e.c_pad)] = dict(samples_per_launch=per, launches_per_call=launches,
                                                   rect_ms=k_r, bank_ms=k_b,
                                                   rect_hbm_share=written / (k_r * 1e-3) / HBM,
                                                   bank_hbm_share=(written + bank_read) / (k_b * 1e-3) / HBM)
        out["predict_%s" % prec] = dict(rect_fwd_per_s=n / (ms_pr * 1e-3), bank_fwd_per_s=n / (ms_pb * 1e-3))
        out["device_bytes_%s" % prec] = dict(fresh=dev0, after_rect=dev1, after_bank=dev2)
        if prec == "bf16":
            for B, S in ((1, 128), (64, 32)):
                x = torch.rand(B, 3, H, H, generator=torch.Generator().manual_seed(1)).to(DEV)
                sel = np.random.RandomState(2).randint(0, n, (B, S))
                rr = PM.gather(table, sel)
                dl = torch.randn(B * S, 1000, generator=torch.Generator().manual_seed(3)).to(DEV)
                ms_er = _host_ms(lambda: (e.eot_forward(x, S, rr), e.eot_backward(dl)), 2)
                ms_eb = _host_ms(lambda: (e.eot_forward(x, S, bank=bank, idx=sel), e.eot_backward(dl)), 2)
                out["eot_fwd_bwd_%dx%d_ms" % (B, S)] = dict(rect=ms_er, bank=ms_eb)
        e.close()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
