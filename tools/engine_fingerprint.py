"""Launch / output fingerprint of the native engine, for comparing two builds of libdorpatch.so.

    python tools/engine_fingerprint.py --lib path/to/libdorpatch.so --out fp.json
    python tools/engine_fingerprint.py --lib A.so --against B.so [--out-dir DIR]   # both, in subprocesses, then diff

(On an H100 one library takes about a minute.  The .npz next to each JSON holds about 40 MB of gradients.)

One run drives every chunk loop of the engine at 112 px, chunk 4, autotune off, for fp32 / tf32 / bf16 and under
the DORPATCH_* variants that change which launches those loops issue.  Two shapes: B = 3 x S = 4 (whole images per
chunk: two lanes everywhere) and B = 2 x S = 5 (images straddle chunks: one lane for dp_attack_grad and
dp_eot_backward).  Per call it records the launch-count delta, the graph-replay counter and the SHA-256 of every
output; a second pass with the engine profiler on (one lane by design) records category -> count, bytes and flops.
The last call reloads a few weights from the device (dp_engine_load_weights_dev: re-standardised convolutions, re-packed
own-stem and fused-GEMM tiles, a GroupNorm whose gamma > 0 flag flips), runs predict / eot_forward / a full parameter
backward on them, and restores the original weights.
Gradients summed with fp32 atomics (the affine / colour EOT adjoint) are not bit-reproducible: they are saved
next to the JSON and compared within the relative L2 bound of tests/test_gpu_eot_xform.py.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, CHUNK, K = 112, 4, 1000
SHAPES = [(3, 4), (2, 5)]
HEAD = ["norm.weight", "norm.bias", "head.fc.weight", "head.fc.bias"]
XFORM_REL_L2 = 1e-5
VARIANTS = [  # (name, environment, precisions)
    ("base", {}, ("fp32", "tf32", "bf16")),
    ("lanes1", {"DORPATCH_LANES": "1"}, ("fp32", "tf32", "bf16")),
    ("graph0", {"DORPATCH_GRAPH": "0"}, ("fp32", "tf32", "bf16")),
    ("k1whole0", {"DORPATCH_K1_WHOLE_MB": "0"}, ("fp32", "tf32", "bf16")),
    ("stembwd_cudnn", {"DORPATCH_STEM_BWD": "cudnn"}, ("bf16",)),   # the fused stem backward exists at bf16 only
    ("fused_gemm", {"DORPATCH_FUSED_GEMM": "1"}, ("bf16",)),       # bf16 only
    ("stem_cudnn", {"DORPATCH_STEM": "cudnn"}, ("bf16",)),          # the library stem at bf16 (padded input)
    ("pool_bwd_fused", {"DORPATCH_POOL_BWD": "fused"}, ("bf16",)),
    ("cpad4", {"DORPATCH_CPAD": "4"}, ("bf16",)),
    ("cpad8", {"DORPATCH_CPAD": "8"}, ("fp32", "tf32")),
]
RELOAD = {  # the "reload" call's changes: name -> new tensor from the original
    "stem.conv.weight": lambda t: t * 1.01,
    "stages.0.blocks.1.conv1.weight": lambda t: t * 1.01,   # no downsample branch: the fused GEMM's operand
    "stages.2.blocks.1.conv2.weight": lambda t: t * 1.01,
    "stages.1.blocks.0.norm2.weight": lambda t: t * t.new_tensor([-1.0] + [1.0] * (t.numel() - 1)),   # gamma > 0 flag flips
    "head.fc.bias": lambda t: t + t.new_tensor(np.linspace(-0.1, 0.1, t.numel(), dtype=np.float32)),
}


def _sha(t):
    import torch
    if isinstance(t, torch.Tensor):
        t = t.detach().contiguous().cpu()
        if t.dtype == torch.bfloat16:
            t = t.view(torch.int16)
        t = t.numpy()
    return hashlib.sha256(np.ascontiguousarray(t).tobytes()).hexdigest()


def _calls(e, B, S, weights):
    """[(name, fn)]: fn() returns {output name: tensor / array}; names ending in '~' are compared within a tolerance."""
    import torch
    from dorpatch_b200 import eot as PE, masks as PM
    from dorpatch_b200.engine import _dev_ptr
    from dorpatch_b200.resnetv2 import param_shapes

    N = B * S
    g = torch.Generator().manual_seed(1000 * B + S)
    img, x, p = (torch.rand(B, 3, H, H, generator=g).cuda() for _ in range(3))
    m = torch.rand(B, 1, H, H, generator=g).cuda()
    dlog = torch.randn(N, K, generator=g).cuda()
    z = torch.randn(CHUNK, 3, H, H, generator=g).cuda()
    dz_logits = torch.randn(CHUNK, K, generator=g).cuda()
    rng = np.random.RandomState(B * 10 + S)
    table = PM.universe(H, 2)
    rects = np.ascontiguousarray(PM.gather(table, rng.randint(0, table.shape[0], (B, S))), np.int16)
    rects_dev = torch.from_numpy(rects.copy()).cuda()
    xf = PE.sample(np.random.RandomState(7 + N), B, S, 0.5, 0.5)
    y = rng.randint(0, K, B)
    tgt = np.array([b % 2 == 0 for b in range(B)])
    G = torch.zeros(B, 3, H, H, device="cuda")
    shapes = param_shapes(K)
    grads = {n: torch.zeros(shapes[n], device="cuda") for n in shapes}
    dt = torch.bfloat16 if e.elem_bytes == 2 else torch.float32
    out_in = torch.empty(N, H, H, e.c_pad, dtype=dt, device="cuda")
    ptr = lambda t: C.c_void_p(t.data_ptr())

    def attack(stage, xforms=None):
        r = e.attack_grad(x, m, p, rects, y, tgt, 0.1, 4.0, stage, G, xforms=xforms)
        out = dict(r)
        out["G~" if xforms is not None else "G"] = G.clone()
        return out

    def eot_fwd(xforms=None):
        return {"logits": e.eot_forward(img, S, rects, xforms=xforms)}

    def params(names, grad_img):
        gi = e.eot_backward_params(dlog, names, [grads[n] for n in names], grad_img=grad_img)
        out = {"grads": torch.cat([grads[n].flatten() for n in names])}
        if gi is not None:
            out["grad_img"] = gi
        return out

    def expand_dev():
        out_in.zero_()
        rc = e.lib.dp_expand_dev(e.handle, _dev_ptr(img), B, S, ptr(rects_dev), ptr(out_in), e._stream())
        assert rc == 0, e.lib.dp_last_error()
        return {"out": out_in.clone()}

    def expand_step_dev():   # reads the clip scale the last dp_attack_grad left
        out_in.zero_()
        rc = e.lib.dp_expand_step_dev(e.handle, _dev_ptr(x), _dev_ptr(m), _dev_ptr(p), B, S, ptr(rects_dev), 1, N - 2,
                                      ptr(out_in), e._stream())
        assert rc == 0, e.lib.dp_last_error()
        return {"out": out_in.clone()}

    def reload():
        e.load_state_dict_dev({n: f(weights[n].clone()).cuda() for n, f in RELOAD.items()})
        try:
            out = dict(zip(("preds", "logits"), e.predict(img, S, rects, return_logits=True)))
            out["eot_logits"] = eot_fwd()["logits"]
            out.update(params(list(shapes), True))
        finally:
            e.load_state_dict_dev({n: weights[n].cuda() for n in RELOAD})
        return out

    calls = [("predict", lambda: dict(zip(("preds", "logits"), e.predict(img, S, rects, return_logits=True))))]
    for stage in (0, 1):
        calls += [("attack_s%d_%d" % (stage, i), lambda stage=stage: attack(stage)) for i in range(4)]
    calls += [
        ("attack_xform", lambda: attack(1, xf)),
        ("expand", lambda: {"out": e.expand(img, S, rects)}),
        ("expand_dev", expand_dev),
        ("expand_step_dev", expand_step_dev),
        ("eot_forward", eot_fwd),
        ("eot_backward_1", lambda: {"grad_img": e.eot_backward(dlog)}),
        ("eot_backward_2", lambda: {"grad_img": e.eot_backward(dlog)}),
        ("eot_forward_xform", lambda: eot_fwd(xf)),
        ("eot_backward_xform", lambda: {"grad_img~": e.eot_backward(dlog)}),
        ("eot_forward_p", eot_fwd),
        ("params_all_img", lambda: params(list(shapes), True)),
        ("params_all", lambda: params(list(shapes), None)),
        ("params_head_img", lambda: params(HEAD, True)),
        ("params_head", lambda: params(HEAD, None)),
        ("net_forward_backward", lambda: dict(zip(("logits", "dz"), e.net_forward_backward(z, dz_logits)))),
        ("reload", reload),
    ]
    return calls


def run(lib_path, out_path):
    import torch
    from dorpatch_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(lib_path)
    from dorpatch_b200.engine import Engine
    from oracle import resnetv2 as OR

    params = OR.random_init(seed=0, affine_jitter=0.1)
    result, arrays = {}, {}
    for vname, env, precisions in VARIANTS:
        for prec in precisions:
            saved = {k: os.environ.get(k) for k in env}
            os.environ.update(env)
            try:
                e = Engine(img=H, precision=prec, chunk=CHUNK, max_images=3, device=0, autotune=False)
            finally:
                for k, v in saved.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
            e.load_state_dict(params)
            for B, S in SHAPES:
                for prof in (False, True):
                    key = "%s/%s/B%dS%d%s" % (vname, prec, B, S, "/prof" if prof else "")
                    rec = result[key] = {}
                    for name, fn in _calls(e, B, S, params):
                        if prof:
                            e.profile(True, reset=True)
                        l0 = e.launch_count
                        outs = fn()
                        torch.cuda.synchronize()
                        r = rec[name] = {"launches": e.launch_count - l0, "graph_replays": e.graph_replays, "out": {}}
                        for k, v in outs.items():
                            if k.endswith("~"):
                                arrays["%s/%s/%s" % (key, name, k)] = v.detach().cpu().numpy()
                                r["out"][k] = list(v.shape)
                            else:
                                r["out"][k] = _sha(v)
                        if prof:
                            r["prof"] = {c: [d["count"], d["bytes"], d["flops"]] for c, d in sorted(e.profile_read().items())}
                    e.profile(False)
            e.close()
            print("done", vname, prec, flush=True)
    with open(out_path, "w") as f:
        json.dump(result, f, indent=1, sort_keys=True)
    np.savez(out_path + ".npz", **arrays)


def diff(a_path, b_path):
    """Number of differences between two runs (printed)."""
    a, b = json.load(open(a_path)), json.load(open(b_path))
    za, zb = np.load(a_path + ".npz"), np.load(b_path + ".npz")
    bad, checked, worst = 0, 0, 0.0
    for key in sorted(set(a) | set(b)):
        if key not in a or key not in b:
            print("MISSING", key); bad += 1; continue
        for call in sorted(set(a[key]) | set(b[key])):
            ra, rb = a[key].get(call), b[key].get(call)
            checked += 1
            if ra != rb:
                print("DIFF", key, call, json.dumps(ra), "!=", json.dumps(rb)); bad += 1
    for k in sorted(set(za.files) | set(zb.files)):
        if k not in za.files or k not in zb.files:
            print("MISSING array", k); bad += 1; continue
        x, y = za[k].astype(np.float64), zb[k].astype(np.float64)
        rel = float(np.linalg.norm(x - y) / (np.linalg.norm(y) + 1e-30))
        worst = max(worst, rel)
        if not rel <= XFORM_REL_L2:
            print("TOL", k, rel); bad += 1
    print("compared %d calls, %d atomics-summed gradients (worst rel L2 %.3g): %d differences"
          % (checked, len(za.files), worst, bad))
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "dorpatch_b200", "lib", "libdorpatch.so"))
    tmp = os.path.join(tempfile.gettempdir(), "engine_fingerprint")
    ap.add_argument("--out", default=os.path.join(tmp, "fingerprint.json"), help="JSON (+ .npz of the atomics-summed gradients)")
    ap.add_argument("--against", help="a second libdorpatch.so: run both in subprocesses and diff")
    ap.add_argument("--out-dir", default=tmp)
    args = ap.parse_args()
    if not args.against:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        run(args.lib, args.out)
        return 0
    os.makedirs(args.out_dir, exist_ok=True)
    outs = []
    for tag, lib in (("a", args.lib), ("b", args.against)):
        out = os.path.join(args.out_dir, "fingerprint_%s.json" % tag)
        t0 = time.time()
        subprocess.run([sys.executable, os.path.abspath(__file__), "--lib", lib, "--out", out], check=True)
        print("%s (%s): %.0f s" % (tag, lib, time.time() - t0), flush=True)
        outs.append(out)
    return 1 if diff(*outs) else 0


if __name__ == "__main__":
    sys.exit(main())
