"""One DorPatch.generate call in a process of its own, for test_gpu_checkpoint.py's fresh-process resume.

    python tests/checkpoint_child.py OUT [--checkpoint PATH --every N] [--cut STAGE,I]

B = 1, 112 px, untargeted, S = 8, dropout 1, 120 iterations per stage, on the fp32 engine with the oracle's random-init
weights.  With --cut the process leaves through SystemExit(3) in place of step (STAGE, I).  OUT receives a pickle of what
the call returned, printed, counted and left in the RNG streams, and the number of lines printed at its last checkpoint
write; it is written on either exit."""
import argparse
import contextlib
import io
import os
import pickle
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dorpatch_b200 import attack as A  # noqa: E402
from dorpatch_b200.engine import Engine  # noqa: E402
from dorpatch_b200.resnetv2 import ResNetV2  # noqa: E402
from dorpatch_b200.utils import NormModel, get_normalize  # noqa: E402
from oracle import resnetv2 as OR  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--checkpoint", default=None)
    ap.add_argument("--every", type=int, default=100)
    ap.add_argument("--cut", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    net = ResNetV2(seed=0)
    net.load_state_dict(OR.random_init(seed=0, affine_jitter=0.1))
    model = torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()
    x = torch.rand(1, 3, 112, 112, generator=torch.Generator().manual_seed(13)).cuda()

    out = dict(cut=False, lines_at_ckpt=0)
    buf = io.StringIO()
    save = A.save_checkpoint

    def counted_save(path, ck):
        save(path, ck)
        out["lines_at_ckpt"] = len(buf.getvalue().splitlines())
    A.save_checkpoint = counted_save

    if args.cut:
        cut = tuple(int(v) for v in args.cut.split(","))
        start = (0, 0)
        if args.checkpoint and os.path.exists(args.checkpoint):
            ck = torch.load(args.checkpoint, weights_only=True)
            start = (int(ck["stage"]), int(ck["i"]))
        grad, calls = Engine.attack_grad, [0, 0]

        def attack_grad(self, *a, **k):
            stage = int(a[8])
            i = (start[1] if stage == start[0] else 0) + calls[stage]
            calls[stage] += 1
            if (stage, i) == cut:
                out["cut"] = True
                raise SystemExit(3)
            return grad(self, *a, **k)
        Engine.attack_grad = attack_grad

    random.seed(1234)
    torch.manual_seed(1234)
    np.random.seed(1234)
    try:
        with contextlib.redirect_stdout(buf):
            gen = A.DorPatch()
            out["m"], out["p"] = gen.generate(model, x, 0.12, 1000, None, 0, max_iterations=120, sampling_size=8,
                                              dropout=1, checkpoint=args.checkpoint, checkpoint_every=args.every)
            out["m"], out["p"] = out["m"].cpu(), out["p"].cpu()
            out["stats"] = gen.last_stats
    finally:
        out["log"] = buf.getvalue().splitlines()
        out["np"], out["torch"] = np.random.get_state(), torch.get_rng_state()
        with open(args.out, "wb") as f:
            pickle.dump(out, f)
        for ent in net._engines.values():
            ent[0].close()


if __name__ == "__main__":
    main()
