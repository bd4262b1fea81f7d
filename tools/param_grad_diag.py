"""How far the engine's parameter gradients are from the oracle, next to how far other implementations of the same
arithmetic are (the yardstick for the bars of tests/test_gpu_param_grad.py).

    python tools/param_grad_diag.py [--out diag.json]

1. fp32, 112 px, B = 4 x S = 8 (the parity test's inputs): per-tensor cosine and overall relative L2 of the engine and
   of the fp32 CPU oracle, both against the fp64 CPU oracle.
2. tf32 / bf16: per-tensor cosine to the fp32 CPU oracle of the engine and of PyTorch-GPU at the same arithmetic, each
   also with the image perturbed by 1e-7 * N(0,1) (below any difference between two implementations): the spread
   of a tensor's cosine under that perturbation is what the statistic can resolve on the random-init network.
3. 10 SGD steps (lr 0.01, cross-entropy, two cutouts, B = 8, 112 px): per step, at the engine's current parameters, the
   loss and gradient of the engine against the fp32 and fp64 oracle restarted from those parameters; then the
   free-running end points: engine vs fp32 oracle, fp32 oracle vs fp64 oracle."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dorpatch_b200 import masks as PM  # noqa: E402
from dorpatch_b200.engine import Engine  # noqa: E402
from oracle import attack as OA  # noqa: E402
from oracle import resnetv2 as OR  # noqa: E402

DEV = "cuda:0"
H = 112


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-300))


def rel_all(g, ref):
    num = sum(float((g[k].double() - ref[k].double()).pow(2).sum()) for k in ref)
    return (num / sum(float(ref[k].double().pow(2).sum()) for k in ref)) ** 0.5


def oracle_grads(params, x01, y, dev="cpu", dtype=torch.float32, autocast=False):
    on = OR.OracleNet({k: v.to(dev, dtype) for k, v in params.items()}, weights_require_grad=True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        logits = on(x01.to(dev, dtype))
    loss = F.cross_entropy(logits.float(), y.to(dev))
    loss.backward()
    return float(loss), {k: p.grad.detach().double().cpu() for k, p in zip(on.keys, on.plist)}


def engine_grads(eng, params, img, rects, S, y):
    names = list(params)
    logits = eng.eot_forward(img.to(DEV), S, rects)
    lg = logits.detach().requires_grad_(True)
    loss = F.cross_entropy(lg, y.to(DEV))
    loss.backward()
    grads = [torch.empty(params[k].shape, device=DEV) for k in names]
    eng.eot_backward_params(lg.grad.contiguous(), names, grads, grad_img=False)
    return float(loss), {k: g.double().cpu() for k, g in zip(names, grads)}


def occluded(img, table, idx, B, S):
    keep = torch.from_numpy(PM.to_bool(table, H)[idx])
    return OA.occlude(img[:, None].double(), keep).reshape(B * S, 3, H, H)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    params = OR.random_init(seed=0, affine_jitter=0.1)
    rep = {}
    B, S = 4, 8
    img = torch.rand((B, 3, H, H), generator=torch.Generator().manual_seed(41))
    table = PM.universe(H, 2)
    idx = np.random.RandomState(42).randint(0, table.shape[0], (B, S))
    rects = PM.gather(table, idx)
    y = torch.tensor([5, 321, 17, 999]).repeat_interleave(S)
    x = occluded(img, table, idx, B, S)
    _, g64 = oracle_grads(params, x, y, dtype=torch.float64)
    _, g32 = oracle_grads(params, x, y)
    eng = Engine(img=H, precision="fp32", chunk=32, max_images=8, autotune=False)
    eng.load_state_dict(params)
    _, gn = engine_grads(eng, params, img, rects, S, y)
    rep["fp32"] = dict(engine_vs_fp64=dict(rel=rel_all(gn, g64), worst_cos=min(cos(gn[k], g64[k]) for k in g64)),
                       oracle32_vs_fp64=dict(rel=rel_all(g32, g64), worst_cos=min(cos(g32[k], g64[k]) for k in g64)),
                       engine_vs_oracle32=dict(rel=rel_all(gn, g32), worst_cos=min(cos(gn[k], g32[k]) for k in g64)))
    print(json.dumps(rep["fp32"]), flush=True)

    noise = [torch.randn(img.shape, generator=torch.Generator().manual_seed(900 + i)) * 1e-7 for i in range(3)]
    for prec in ("tf32", "bf16"):
        e = Engine(img=H, precision=prec, chunk=32, max_images=8, autotune=False)
        e.load_state_dict(params)
        old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = prec == "tf32"
        torch.backends.cuda.matmul.allow_tf32 = prec == "tf32"
        nat, tch = [], []
        for nz in [torch.zeros_like(img)] + noise:
            im = (img + nz).clamp(0, 1)
            nat.append(engine_grads(e, params, im, rects, S, y)[1])
            tch.append(oracle_grads(params, occluded(im, table, idx, B, S).float(), y, dev=DEV, autocast=prec == "bf16")[1])
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        e.close()
        per = {}
        for k in g32:
            cn = [cos(g[k], g32[k]) for g in nat]
            ct = [cos(g[k], g32[k]) for g in tch]
            per[k] = dict(native=cn[0], torch=ct[0], native_spread=max(cn) - min(cn), torch_spread=max(ct) - min(ct),
                          native_min=min(cn), torch_max=max(ct))
        worst = sorted(per.items(), key=lambda kv: kv[1]["native"] - kv[1]["torch"])[:6]
        rep[prec] = dict(worst=worst, max_torch_spread=max(v["torch_spread"] for v in per.values()),
                         max_native_spread=max(v["native_spread"] for v in per.values()),
                         n_below_torch_minus_001=sum(v["native"] < v["torch"] - 0.01 for v in per.values()),
                         n_native_max_below_torch_min_minus_001=sum(
                             max(cos(g[k], g32[k]) for g in nat) < min(cos(g[k], g32[k]) for g in tch) - 0.01 for k in g32))
        print(prec, json.dumps({k: v for k, v in rep[prec].items() if k != "worst"}), flush=True)
        for k, v in worst:
            print("  ", k, json.dumps(v), flush=True)

    # SGD
    Bs, steps, lr = 8, 10, 0.01
    rs = np.random.RandomState(121)
    pn = {k: v.clone() for k, v in params.items()}          # engine's trajectory
    p32 = {k: v.clone() for k, v in params.items()}         # free-running fp32 oracle
    p64 = {k: v.double().clone() for k, v in params.items()}  # free-running fp64 oracle
    e = Engine(img=H, precision="fp32", chunk=8, max_images=8, autotune=False)
    e.load_state_dict(pn)
    rows = []
    for it in range(steps):
        im = torch.rand((Bs, 3, H, H), generator=torch.Generator().manual_seed(200 + it))
        yy = torch.from_numpy(rs.randint(0, 1000, Bs))
        rc = np.zeros((Bs, 1, 4, 4), np.int16)
        keep = torch.ones(Bs, 1, 1, H, H, dtype=torch.bool)
        for b in range(Bs):
            for r in range(2):
                s = rs.randint(16, 48)
                r0, c0 = rs.randint(0, H - s), rs.randint(0, H - s)
                rc[b, 0, r] = (r0, r0 + s, c0, c0 + s)
                keep[b, 0, 0, r0:r0 + s, c0:c0 + s] = False
        xo = OA.occlude(im[:, None].double(), keep).reshape(Bs, 3, H, H)
        ln, gn_ = engine_grads(e, pn, im, rc, 1, yy)
        lo32, go32 = oracle_grads(pn, xo.float(), yy)
        lo64, go64 = oracle_grads(pn, xo, yy, dtype=torch.float64)
        lf32, gf32 = oracle_grads(p32, xo.float(), yy)
        lf64, gf64 = oracle_grads(p64, xo, yy, dtype=torch.float64)
        step_norm = (sum(float(v.double().pow(2).sum()) for v in go64.values()) ** 0.5) * lr
        pnorm = sum(float(v.double().pow(2).sum()) for v in pn.values()) ** 0.5
        rows.append(dict(step=it, loss_engine_vs_oracle32_same_params=abs(ln - lo32) / abs(lo32),
                         grad_engine_vs_fp64_same_params=rel_all(gn_, go64), grad_oracle32_vs_fp64_same_params=rel_all(go32, go64),
                         update_over_params=step_norm / pnorm,
                         loss_free_oracle32_vs_free_fp64=abs(lf32 - lf64) / abs(lf64)))
        print(json.dumps(rows[-1]), flush=True)
        for k in pn:
            pn[k] = pn[k] - lr * gn_[k].float()
            p32[k] = p32[k] - lr * gf32[k].float()
            p64[k] = p64[k] - lr * gf64[k]
        e.load_state_dict_dev({k: v.to(DEV) for k, v in pn.items()})
    e.close()
    rep["sgd"] = dict(steps=rows, final_engine_vs_oracle32=rel_all(pn, p32), final_oracle32_vs_fp64=rel_all(p32, p64),
                      final_engine_vs_fp64=rel_all(pn, p64))
    print(json.dumps({k: v for k, v in rep["sgd"].items() if k != "steps"}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
