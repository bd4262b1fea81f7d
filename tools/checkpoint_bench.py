"""Cost of generate()'s step-level checkpoints against one step, one JSON line per universe.

    python tools/checkpoint_bench.py [--B 64] [--S 128] [--precision tf32] [--every 3]

On a random-init ResNetV2-50x1-BiT at 224 px, B images x S EOT samples, host sampler, per universe (one-patch dropout 2:
2 520 masks; two-patch dropout 1: 2 520 masks).  A first generate() call writes a checkpoint after every `every`-th
step and is cut (an exception in place of the step) at step 2 * every + 1; a second call resumes from the file and is
cut one step later.  Reported:
  step_s        median host-clock time between consecutive steps' gradient calls (each returns host results, so each
                interval ends in a device synchronise), over the steps that neither scan the universe nor write;
  write_s       the second write: the snapshot (device-to-host copies, one failed-set read per image) and the atomic
                file write with fsync, after a device synchronise; failed_read_s is its failed-set reads alone;
  load_s        reading and validating the file at resume (read_checkpoint);
  file_mb       the checkpoint's size.
The checkpoint goes to a temporary directory, removed at the end.  Library algorithms come from the heuristics
(DORPATCH_AUTOTUNE=0).  The GPU's name and power limit are read in the same process.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("DORPATCH_AUTOTUNE", "0")
from dorpatch_b200 import attack as A                 # noqa: E402
from dorpatch_b200.engine import Engine               # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2           # noqa: E402
from dorpatch_b200.utils import NormModel, get_normalize  # noqa: E402
from tools.pc_bench import gpu_info                   # noqa: E402

IMG = 224
UNIVERSES = {"one_patch_dropout2": dict(dropout=2, pc_n_patch=1), "two_patch_dropout1": dict(dropout=1, pc_n_patch=2)}


class _Cut(Exception):
    pass


def timed_call(model, x, kw, path, every, cut):
    """generate() until step `cut` of stage 0; returns the gradient calls' start times and the writes' / loads' times."""
    t = dict(grad=[], write=[], read_failed=[], load=[])
    grad, write, read, fread = Engine.attack_grad, A.write_checkpoint, A.read_checkpoint, Engine.failed_read
    calls = [0]

    def attack_grad(self, *a, **k):
        t["grad"].append(time.perf_counter())
        if calls[0] == cut:
            raise _Cut()
        calls[0] += 1
        return grad(self, *a, **k)

    def write_checkpoint(*a, **k):
        torch.cuda.synchronize()
        t["read_failed"].append(0.0)
        t0 = time.perf_counter()
        write(*a, **k)
        t["write"].append((t0, time.perf_counter() - t0))

    def failed_read(self, b):
        t0 = time.perf_counter()
        r = fread(self, b)
        if t["read_failed"]:
            t["read_failed"][-1] += time.perf_counter() - t0
        return r

    def read_checkpoint(*a, **k):
        t0 = time.perf_counter()
        r = read(*a, **k)
        t["load"].append(time.perf_counter() - t0)
        return r

    Engine.attack_grad, A.write_checkpoint, A.read_checkpoint, Engine.failed_read = \
        attack_grad, write_checkpoint, read_checkpoint, failed_read
    np.random.seed(1234)
    torch.manual_seed(1234)
    try:
        A.DorPatch().generate(model, x, 0.12, 1000, None, 0, sampling_size=kw.pop("S"), checkpoint=path,
                              checkpoint_every=every, **kw)
    except _Cut:
        pass
    finally:
        Engine.attack_grad, A.write_checkpoint, A.read_checkpoint, Engine.failed_read = grad, write, read, fread
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--S", type=int, default=128)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--every", type=int, default=3)
    args = ap.parse_args()
    os.environ["DORPATCH_PRECISION"] = args.precision
    torch.cuda.set_device(0)
    net = ResNetV2(seed=0)
    model = torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()
    x = torch.rand(args.B, 3, IMG, IMG, generator=torch.Generator().manual_seed(0)).cuda()
    info = gpu_info(0)
    tmp = tempfile.mkdtemp(prefix="dorpatch_ckpt_bench_")
    try:
        for name, uni in UNIVERSES.items():
            path = os.path.join(tmp, "adv_ckpt_0.pt")
            kw = dict(uni, S=args.S, max_iterations=5000)
            first = timed_call(model, x, dict(kw), path, args.every, 2 * args.every + 1)
            size = os.path.getsize(path)
            second = timed_call(model, x, dict(kw), path, args.every, 1)
            os.remove(path)
            g = first["grad"]
            w0, w = first["write"][-1]
            steps = [b - a for a, b in zip(g[1:-1], g[2:])                          # step 0 scans the universe
                     if not any(a <= t0 < b for t0, _ in first["write"])]
            step = float(np.median(steps))
            print(json.dumps(dict(
                universe=name, B=args.B, S=args.S, img=IMG, precision=args.precision, step_s=round(step, 4),
                steps_timed=len(steps), write_s=round(w, 4), failed_read_s=round(first["read_failed"][-1], 4),
                load_s=round(second["load"][0], 4), file_mb=round(size / 2 ** 20, 1),
                write_over_step=round(w / step, 4), load_over_step=round(second["load"][0] / step, 4), gpu=info)),
                flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        for ent in net._engines.values():
            ent[0].close()


if __name__ == "__main__":
    main()
