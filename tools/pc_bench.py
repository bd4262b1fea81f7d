"""PatchCleanser evaluation cost per image on one GPU, one-patch vs two-patch window, one JSON line.

    python tools/pc_bench.py [--images K] [--precisions tf32,bf16]

K synthetic 224 px images go through adv_x = paste(x, mask, pattern, eps) and then, for n_patch 1 and 2, through
PatchCleanser(MaskWindow(224, r, n_patch), model).robust_predict(adv_x, True) at the four ratios -- exactly the
evaluation main.py runs per image -- on a random-init ResNetV2-50x1-BiT.  Per precision and n_patch it reports the
seconds per image, the masked forwards per image counted from the records (round 1 + round 2 + certificate) and their
rate; as the yardstick for that rate, a plain dp_predict over the 2520-mask universe on the same engine.  Every shape is
warmed up on an extra image first.  The GPU's name and power limit are read in the same process.

    torchrun --nproc-per-node N tools/pc_bench.py [...]

runs the same evaluation with the masked forwards sharded over N GPUs (every rank gets the single-GPU records); rank 0
prints the line, with the world size, every rank's GPU name and power limit, and per window the masked forwards each
rank ran.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dorpatch_b200 import masks as PM                                    # noqa: E402
from dorpatch_b200.defenses.PatchCleanser import MaskWindow, PatchCleanser  # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2                               # noqa: E402
from dorpatch_b200.utils import NormModel, get_normalize                  # noqa: E402

IMG = 224
RATIOS = (0.015, 0.03, 0.06, 0.12)


def gpu_info(dev=0):
    info = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_mhz"] = float(q[0]), float(q[1])
    except Exception as ex:            # the figures stay usable without it; the line says why the field is missing
        info["power_limit_error"] = repr(ex)[:200]
    return info


def forwards(rec):
    """Masked forwards robust_predict ran for this record: round 1, one round-1-sized call per mask whose label is not the
    majority (PatchCleanser.py:80-90; the majority as :74-75 picks it), the certificate."""
    p1 = torch.from_numpy(np.asarray(rec.preds_1))
    labels, counts = p1.unique(sorted=False, return_counts=True)
    majority = labels[counts.argmax()].item()
    round2 = int((p1 != majority).sum()) * len(p1) if len(labels) > 1 else 0
    return len(p1), round2, len(rec.preds_2)


def evaluate(defs, images, dist=None):
    torch.cuda.synchronize()
    if dist:
        dist.barrier()                           # every rank starts the timed window together
    t0 = time.perf_counter()
    recs = [[d.robust_predict(im, True) for d in defs] for im in images]
    torch.cuda.synchronize()                     # dp_predict already ends in a stream synchronise; this makes it explicit
    return time.perf_counter() - t0, recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=2)
    ap.add_argument("--precisions", default="tf32,bf16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/pc_bench.py needs a CUDA device (H100)")
    dist, rank, world = None, 0, 1
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:     # torchrun: one process per GPU, robust_predict shards over them
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        rank, world = dist.get_rank(), dist.get_world_size()
    K = args.images
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(K + 1, 3, IMG, IMG, generator=g).cuda()
    mask = (torch.rand(K + 1, 1, IMG, IMG, generator=g) < 0.12).float().cuda()      # 12 % patch budget, scattered pixels
    pattern = torch.rand(K + 1, 3, IMG, IMG, generator=g).cuda()
    net = ResNetV2(seed=0)
    model = torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2")))
    uni = PM.gather(PM.universe(IMG, 2), np.arange(2520))
    out = {"tool": "pc_bench", "img": IMG, "images": K, "ratios": list(RATIOS), "model": "ResNetV2-50x1-BiT random-init (seed 0)",
           "gpu": gpu_info(local), "legs": {}}
    if dist:
        out["world"] = world
        out["gpus"] = [None] * world
        dist.all_gather_object(out["gpus"], out["gpu"])
    for prec in args.precisions.split(","):
        os.environ["DORPATCH_PRECISION"] = prec          # the engine PatchCleanser asks the model for
        eng = net.engine(IMG, max_images=K + 1)
        adv, _, _ = eng.paste(x, mask, pattern, 4.0)
        leg = {"chunk": eng.chunk}
        for n_patch in (1, 2):
            with contextlib.redirect_stdout(io.StringIO()):
                defs = [PatchCleanser(MaskWindow(IMG, r, n_patch), model, shard=True) for r in RATIOS]
            evaluate(defs, adv[K:], dist)                                       # warm-up image: every call shape once
            ran0 = sum(d.forwards for d in defs)
            dt, recs = evaluate(defs, adv[:K], dist)
            n = np.array([[forwards(r) for r in row] for row in recs])          # [K, ratios, (round 1, round 2, certificate)]
            per_img = n.sum(axis=(1, 2))
            leg["n_patch_%d" % n_patch] = {
                "s_per_image": dt / K, "forwards_per_image": float(per_img.mean()),
                "forwards_per_image_by_round": dict(zip(("round1", "round2", "certificate"), n.sum(axis=1).mean(0).tolist())),
                "forwards_per_s": float(per_img.sum()) / dt,
                "certified": [[bool(r.certification) for r in row] for row in recs]}
            if dist:
                ran = [None] * world                                            # masked forwards each rank ran per image
                dist.all_gather_object(ran, (sum(d.forwards for d in defs) - ran0) / K)
                leg["n_patch_%d" % n_patch]["forwards_per_image_by_rank"] = ran
        img0 = x[:1].contiguous()
        eng.predict(img0, 2520, uni)
        ts = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.predict(img0, 2520, uni)
            ts.append(time.perf_counter() - t0)
        leg["dp_predict_2520"] = {"forwards_per_s": 2520 / float(np.median(ts)), "ms": float(np.median(ts)) * 1e3,
                                  "note": "one image x the 2520-mask universe through dp_predict, median of 5"}
        for n_patch in (1, 2):
            leg["n_patch_%d" % n_patch]["rate_vs_dp_predict"] = (leg["n_patch_%d" % n_patch]["forwards_per_s"]
                                                                 / leg["dp_predict_2520"]["forwards_per_s"])
        out["legs"][prec] = leg
        eng.close()
        net._engines.clear()
    if rank == 0:
        print(json.dumps(out))
    if dist:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
