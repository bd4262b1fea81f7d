"""The kernels of the attack's own arithmetic, op by op against their restatements in oracle/attack.py, at every image
size from 56 to 336 px:

- K4 (CW loss, argmax, dlogits) bit for bit against oracle.attack.cw_loss, torch.argmax and torch autograd, on rows
  built where such kernels go wrong: the association order of the margin, the ReLU gate at exactly zero, ties, the
  -1e4 label slot, inf and NaN;
- the structural loss and its one-sided gradient dLs against fp64 autograd of oracle.attack.struct_loss;
- K3's pattern path (chain rule through the clipped paste, bias, sign step, clip) against fp64 autograd;
- K1^T, the masked EOT reduce of the fp32 / tf32 engines and of the bf16 engine's cuDNN stem-backward end, against an
  fp64 sum, over more than one 128-sample pass of its loop and from the middle of an image.

Outputs are filled with NaN (or a sentinel) first, so an element a kernel leaves unwritten cannot pass."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import attack as OA
from test_gpu_occlusion import _engine, _occluded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [56, 112, 168, 224, 280, 336]
CPAD = {"fp32": 4, "tf32": 4, "bf16": 8}      # channels per pixel of d(input) the engines pick (DORPATCH_CPAD unset)
# one object per engine configuration, shared by every parametrisation below, so that pytest groups the tests of one
# engine and holds one engine at a time
_CFG = {(p, H): (p, H) for p in CPAD for H in SIZES}


def _engines(precisions, sizes=SIZES):
    cfgs = [_CFG[(p, H)] for p in precisions for H in sizes]
    return pytest.mark.parametrize("eng", cfgs, indirect=True, ids=["%s-%d" % c for c in cfgs])


@pytest.fixture(scope="module")
def eng(request, oracle_params):
    """The engine of one (precision, size), closed when pytest moves on to the next.  The bf16 engine runs its cuDNN
    stem-backward end, the one that ends in K1^T."""
    precision, H = request.param
    env = {"DORPATCH_STEM_BWD": "cudnn"} if precision == "bf16" else {}
    e = _engine(oracle_params, precision, img=H, chunk=2, max_images=2, **env)
    yield e
    e.close()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _check(rc):
    from dorpatch_b200 import _lib
    _lib.check(rc)


# ---------------------------------------------------------------------------------------------------------------------
# K4
# ---------------------------------------------------------------------------------------------------------------------
def _cw_rows(K, conf, seed, R=257):
    """R rows of fp32 logits [R,K], labels [R], targeted flags [R] and a name per row: first the rows built on purpose,
    then random rows at logit scales 1, 5 and 20."""
    rng = np.random.RandomState(seed)
    f32, c = np.float32, np.float32(conf)
    rows, ys, tgs, names = [], [], [], []

    def add(name, row, y, tg):
        rows.append(np.asarray(row, f32)); ys.append(int(y)); tgs.append(bool(tg)); names.append(name)

    def below(v):
        """a row whose entries are all below v"""
        return (v - 1 - np.abs(rng.randn(K)) * 5).astype(f32)

    def margin_row(name, r, o, tg):
        """label logit r, largest other logit o at a random index, every other logit below o"""
        y, j = rng.choice(K, 2, replace=False)
        row = below(o)
        row[y], row[j] = r, o
        add(name, row, y, tg)

    # the two association orders: the reference's (c + other) - real against c + (other - real), searched in float32
    r = (rng.randn(400000) * 20).astype(f32)
    for tg in (True, False):
        o = (rng.randn(400000) * 20).astype(f32)
        ref = (c + o) - r if tg else (c + r) - o
        old = c + (o - r) if tg else c + (r - o)
        hit = np.nonzero((np.maximum(ref, 0) != np.maximum(old, 0)))[0][:6]
        assert conf == 0 or len(hit) == 6
        for i in hit:
            margin_row("order-value", r[i], o[i], tg)
        # pre within a few ulps of 0: the orders disagree on its sign (and so on the gate)
        base = (r - c) if tg else (r + c)
        o = (base + rng.randint(-4, 5, r.shape) * np.spacing(base)).astype(f32)
        ref = (c + o) - r if tg else (c + r) - o
        old = c + (o - r) if tg else c + (r - o)
        hit = np.nonzero((ref >= 0) != (old >= 0))[0][:6]
        assert conf == 0 or len(hit) == 6
        for i in hit:
            margin_row("order-sign", r[i], o[i], tg)
        # pre exactly 0: the gate passes
        for _ in range(3):
            v = f32(rng.randn() * 20)
            if tg:
                margin_row("pre-zero", f32(c + v), v, tg)        # (c + other) - real == 0
            else:
                margin_row("pre-zero", v, f32(c + v), tg)        # (c + real) - other == 0
    # ties between non-label classes, in different lanes and (K > 32) in the same lane; the lowest index takes the gradient
    pairs = [(3, 7), (1, K - 1)] + ([(5, 37)] if K > 37 else []) + ([(31, 32)] if K > 32 else [])
    for i1, i2 in pairs:
        for tg in (True, False):
            row = below(10.0)
            row[i1] = row[i2] = f32(10.0)
            y = next(k for k in range(K) if k not in (i1, i2))
            row[y] = f32(9.5)
            add("tie-other", row, y, tg)
    # a tie for the row maximum between the label and another class, the label first and the label last
    for y, j in ((0, 4), (K - 1, 2)):
        for tg in (True, False):
            row = below(3.0)
            row[y] = row[j] = f32(3.0)
            add("tie-label", row, y, tg)
    # the label as the row maximum
    for tg in (True, False):
        y = rng.randint(K)
        row = below(0.0)
        row[y] = f32(4.0)
        add("label-max", row, y, tg)
    # every other logit <= -1e4: the -1e4 label slot wins (no gradient to another class), or ties with index 0 / K-1
    for tg, lab in ((True, -2e4), (False, 3.0)):
        y = rng.randint(K)
        row = (-1e4 - 1 - np.abs(rng.randn(K)) * 100).astype(f32)
        row[y] = f32(lab)
        add("label-slot", row, y, tg)
        for y in (0, K - 1):
            row = np.full(K, -1e4, f32)
            row[y] = f32(lab)
            add("label-slot-tie", row, y, tg)
    # non-finite logits: any of them makes the reference's real = sum(l * onehot) NaN (0 * inf = NaN)
    inf, nan = np.inf, np.nan
    for name, vals in (("+inf", {2: inf}), ("-inf", {2: -inf}), ("+inf-label", {"y": inf}), ("-inf-label", {"y": -inf}),
                       ("nan", {3: nan}), ("nan-label", {"y": nan}), ("nan-and-inf", {1: inf, K - 2: nan, 4: nan})):
        for tg in (True, False):
            y = 5
            row = (rng.randn(K) * 5).astype(f32)
            for k, v in vals.items():
                row[y if k == "y" else k] = v
            add(name, row, y, tg)
    for name, v in (("all--inf", -inf), ("all-nan", nan), ("all-+inf", inf)):
        for tg in (True, False):
            add(name, np.full(K, v, f32), rng.randint(K), tg)
    assert len(rows) < R
    while len(rows) < R:
        add("random", (rng.randn(K) * [1, 5, 20][len(rows) % 3]).astype(f32), rng.randint(K), rng.rand() < 0.5)
    return torch.from_numpy(np.stack(rows)), torch.tensor(ys), torch.tensor(tgs), np.array(names)


def _cw_ref(logits, y, tg, conf, inv_s):
    """oracle.attack.cw_loss of every row (the targeted rows as one batch, the untargeted as another), the torch autograd
    gradient of (inv_s * loss).sum() with respect to the logits, and torch.argmax."""
    lg = logits.clone().requires_grad_(True)
    loss = torch.empty(len(y))
    total = 0
    for t in (True, False):
        rows = torch.nonzero(tg == t).flatten()
        if len(rows):
            part = OA.cw_loss(lg[rows], y[rows], lg.shape[1], t, conf)
            loss[rows] = part.detach()
            total = total + (inv_s * part).sum()
    total.backward()
    return loss, lg.grad, logits.argmax(1)


def _cw_gpu(e, logits, y, tg, conf, inv_s):
    N, K = logits.shape
    ld = logits.to(DEV)
    loss = torch.full((N,), 7.0, device=DEV)
    preds = torch.full((N,), -5, dtype=torch.int32, device=DEV)
    dl = torch.full((N, K), 3.0, device=DEV)
    yd, td = y.to(torch.int32).to(DEV), tg.to(torch.uint8).to(DEV)
    _check(e.lib.dp_debug_cw(e.handle, _ptr(ld), _ptr(yd), _ptr(td), conf, inv_s, _ptr(loss), _ptr(preds), _ptr(dl),
                             N, K, e._stream()))
    am = torch.full((N,), -5, dtype=torch.int32, device=DEV)
    _check(e.lib.dp_debug_cw(e.handle, _ptr(ld), None, None, 0.0, 0.0, None, _ptr(am), None, N, K, e._stream()))
    torch.cuda.synchronize()
    return loss.cpu(), preds.cpu().long(), dl.cpu(), am.cpu().long()


@_engines(["fp32"], [56])
@pytest.mark.parametrize("conf", [0.0, 0.1, 5.0])
@pytest.mark.parametrize("K", [10, 31, 32, 33, 1000])
def test_cw_kernel_bit_exact(eng, K, conf):
    """K4 against the reference bit for bit: loss equal (NaN where torch gives NaN), preds (with and without labels)
    equal to torch.argmax, dlogits equal to the autograd gradient of (inv_s * cw_loss).sum(), inv_s = float32 1 / S.
    N = 1, 7, 9 and 257 rows (warp-per-sample tails), targeted and untargeted rows mixed."""
    logits, y, tg, names = _cw_rows(K, conf, seed=K * 7 + int(conf * 10))
    bad = {}
    for off, N, S in ((0, 257, 128), (0, 1, 1), (40, 7, 7), (100, 9, 3)):
        inv_s = float(np.float32(1) / np.float32(S))
        sl = slice(off, off + N)
        loss_r, d_r, am_r = _cw_ref(logits[sl], y[sl], tg[sl], conf, inv_s)
        loss, preds, d, am = _cw_gpu(eng, logits[sl], y[sl], tg[sl], conf, inv_s)
        nan = torch.isnan(loss_r)
        checks = {
            "loss": (torch.isnan(loss) != nan) | (~nan & (loss != loss_r)),
            "preds": preds != am_r,
            "argmax": am != am_r,
            "dlogits": (d != d_r).any(1),
        }
        for what, wrong in checks.items():
            for i in torch.nonzero(wrong).flatten().tolist():
                bad.setdefault(what, set()).add(names[off + i])
    assert not bad, "rows that differ from the reference: %s" % {k: sorted(v) for k, v in bad.items()}


@_engines(["fp32"], [56])
def test_attack_op_hooks_refuse_bad_arguments(eng):
    """dp_debug_cw refuses a label outside [0, K) and a loss without its flags or an argmax without preds;
    dp_debug_reduce refuses samples outside [0, B*S)."""
    from dorpatch_b200 import _lib
    lg = torch.zeros(2, 10, device=DEV)
    td = torch.zeros(2, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, device=DEV)
    for y in ([0, 10], [-1, 0]):
        yd = torch.tensor(y, dtype=torch.int32, device=DEV)
        assert eng.lib.dp_debug_cw(eng.handle, _ptr(lg), _ptr(yd), _ptr(td), 0.0, 1.0, _ptr(out), None, None, 2, 10,
                                 eng._stream()) == 1
        assert b"outside [0, 10)" in _lib.load().dp_last_error()
    yd = torch.zeros(2, dtype=torch.int32, device=DEV)
    assert eng.lib.dp_debug_cw(eng.handle, _ptr(lg), _ptr(yd), None, 0.0, 1.0, _ptr(out), None, None, 2, 10, eng._stream()) == 1
    assert eng.lib.dp_debug_cw(eng.handle, _ptr(lg), None, None, 0.0, 1.0, None, None, None, 2, 10, eng._stream()) == 1
    assert eng.lib.dp_debug_reduce(eng.handle, _ptr(lg), None, None, 0, None, 2, 1, 1, 2, _ptr(out), eng._stream()) == 1


# ---------------------------------------------------------------------------------------------------------------------
# structural loss and K3
# ---------------------------------------------------------------------------------------------------------------------
def _attack_grad(e, x, m, p, eps, stage):
    """attack_grad of B = 2 images with one unoccluded sample each (its paste and struct kernels are what these tests
    read): the host results and the paste scale, min(eps / l2, 1) in float32 as the paste kernel forms it."""
    B, H = x.shape[0], x.shape[-1]
    G = torch.empty(B, 3, H, H, device=DEV)
    r = e.attack_grad(x, m, p, np.zeros((B, 1, 4, 4), np.int16), np.array([1, 2]), [True, False], 0.1, eps, stage, G)
    torch.cuda.synchronize()
    return r, np.minimum(np.float32(eps) / r["l2"], np.float32(1))


def _adv32(x, m, p, sc):
    """x + (m * (p - x)) * scale in float32: the paste kernel's arithmetic."""
    return x + (m * (p - x)) * torch.from_numpy(sc).view(-1, 1, 1, 1)


def _update(e, x, m, p, G, lr, structured, stage, clip=(0.0, 1.0), bias=None):
    """attack_update on copies of m and p: (grad_pattern_out, updated pattern, updated mask), on the CPU."""
    B = x.shape[0]
    md, pd = m.clone(), p.clone()
    gp = torch.full_like(p, float("nan"))
    gm = torch.full_like(m, float("nan")) if stage == 0 else None
    e.attack_update(x, md, pd, G, np.full(B, lr, np.float32), np.full(B, structured, np.float32), np.full(B, 1e-5),
                    1e-3, stage, clip_min=clip[0], clip_max=clip[1], grad_pattern_out=gp, grad_mask_out=gm,
                    grad_pattern_bias=bias)
    torch.cuda.synchronize()
    return gp.cpu(), pd.cpu(), md.cpu()


def _struct_inputs(kind, H, seed):
    """x, p [2,3,H,H]: random; quantised to k/16 (ties lr == ud and zero differences are frequent, and exact in fp32 and
    fp64); or random with flat regions in x (local variance 0, weight 1e5), different in each image."""
    g = torch.Generator().manual_seed(seed)
    if kind == "quantised":
        x, p = (torch.randint(0, 17, (2, 3, H, H), generator=g) / 16.0 for _ in range(2))
    else:
        x, p = torch.rand(2, 3, H, H, generator=g), torch.rand(2, 3, H, H, generator=g)
    if kind == "flat":
        x[0, :, : H // 2] = 0.5
        x[1, :, H // 4: H // 2, H // 3:] = 0.25
    return x, p


def _sign_and_value_errors(got, ref):
    """elements outside |got - ref| <= 1e-5 |ref| + 1e-6 max |ref|"""
    got = got.double()
    return int(((got - ref).abs() > 1e-5 * ref.abs() + 1e-6 * ref.abs().max()).sum())


@_engines(["fp32"])
@pytest.mark.parametrize("kind", ["random", "quantised", "flat"])
def test_struct_loss_and_gradient_vs_fp64(eng, kind):
    """The struct kernel's loss and dLs (quirk Q4's one-sided gradient) against fp64 autograd of
    oracle.attack.struct_loss.  m = 1 and a large eps make paste's scale exactly 1, so adv = x + (p - x) in fp32, which
    the reference builds the same way before it promotes to fp64; then attack_update(G = 0, structured = 1, lr = 0)
    writes grad_pattern_out = dLs exactly.  Loss: relative 1e-5; dLs: |got - ref| <= 1e-5 |ref| + 1e-6 max |ref|; on the
    quantised inputs also every exact zero and every sign.  (There the two one-sided terms of a pixel can cancel exactly;
    fp64 autograd, which forms them along different paths, leaves residues near 1e-16 of the largest value, which count
    as zero.)"""
    H = eng.img
    x, p = _struct_inputs(kind, H, seed=H * 3 + len(kind))
    m = torch.ones(2, 1, H, H)
    xd, md, pd = x.to(DEV), m.to(DEV), p.to(DEV)
    r, sc = _attack_grad(eng, xd, md, pd, 1e4, stage=1)
    assert (sc == 1).all()
    gp, p_after, _ = _update(eng, xd, md, pd, torch.zeros_like(xd), 0.0, 1.0, stage=1)
    assert torch.equal(p_after, p)
    adv32 = _adv32(x, m, p, sc)
    if kind == "quantised":
        assert torch.equal(adv32, p)
    adv = adv32.double().requires_grad_(True)
    loss = OA.struct_loss(adv, OA.local_variance(x.double())[0].mean(1))
    loss.sum().backward()
    ref = adv.grad
    rel = np.abs(r["loss_struc"] - loss.detach().numpy()) / loss.detach().numpy()
    nbad = _sign_and_value_errors(gp, ref)
    print("struct %s H=%d: loss rel %s, dLs max |err| / max |ref| %.2e" % (
        kind, H, rel, float((gp.double() - ref).abs().max() / ref.abs().max())))
    assert (rel <= 1e-5).all(), rel
    assert torch.isfinite(gp).all() and nbad == 0, "dLs: %d elements outside the bound" % nbad
    if kind == "quantised":
        ref = torch.where(ref.abs() <= 1e-12 * ref.abs().max(), torch.zeros_like(ref), ref)
        assert (ref == 0).any() and torch.equal(gp == 0, ref == 0)
        assert torch.equal(torch.sign(gp.double()), torch.sign(ref))


@_engines(["fp32"])
@pytest.mark.parametrize("stage", [0, 1])
def test_update_pattern_path_vs_fp64(eng, stage):
    """K3's pattern path, gp = m c (G + structured dLs) + bias, against fp64 autograd of <G, adv> + structured *
    struct_loss(adv) with respect to the pattern, adv = x + clip_paste(m, p, x, eps) with the scale detached, plus the
    bias.  Paste's scale < 1 on both images; G and structured chosen so that both terms have comparable size.  With
    lr = 0 the pattern (and the mask) stay untouched; with lr > 0 and the clip range [0.2, 0.7] the pattern is exactly
    clamp(p - lr sign(gp), 0.2, 0.7).  gp: |got - ref| <= 1e-5 |ref| + 1e-6 max |ref|, and sign(got) == sign(ref) wherever
    |ref| > 1e-5 max |ref|."""
    H = eng.img
    g = torch.Generator().manual_seed(H * 5 + stage)
    x, p, m = torch.rand(2, 3, H, H, generator=g), torch.rand(2, 3, H, H, generator=g), torch.rand(2, 1, H, H, generator=g)
    eps = 0.6 * float((m * (p - x)).flatten(1).norm(dim=1).min())
    xd, md, pd = x.to(DEV), m.to(DEV), p.to(DEV)
    _, sc = _attack_grad(eng, xd, md, pd, eps, stage)
    assert (sc < 1).all()
    adv32 = _adv32(x, m, p, sc).double()
    lvx = OA.local_variance(x.double())[0].mean(1)
    a = adv32.clone().requires_grad_(True)
    OA.struct_loss(a, lvx).sum().backward()
    structured = 0.37
    G = torch.randn(2, 3, H, H, generator=g) * (structured * float(a.grad.abs().mean()))
    p64 = p.double().requires_grad_(True)
    delta = OA.clip_paste(m.double(), p64, x.double(), eps)
    adv = adv32 + (delta - delta.detach())            # the kernels' value of adv, the reference's derivative
    ((G.double() * adv).sum() + structured * OA.struct_loss(adv, lvx).sum()).backward()
    bias = torch.randn(2, 3, H, H, generator=g) * (0.5 * float(p64.grad.abs().mean()))
    ref = p64.grad + bias.double()
    Gd, bd = G.to(DEV), bias.to(DEV)
    gp0, p0, m0 = _update(eng, xd, md, pd, Gd, 0.0, structured, stage, (0.2, 0.7), bd)
    assert torch.equal(p0, p) and torch.equal(m0, m)
    lr = 0.05
    gp, p1, _ = _update(eng, xd, md, pd, Gd, lr, structured, stage, (0.2, 0.7), bd)
    assert torch.equal(gp, gp0)
    nbad = _sign_and_value_errors(gp, ref)
    big = ref.abs() > 1e-5 * ref.abs().max()
    nsign = int((torch.sign(gp.double()) != torch.sign(ref))[big].sum())
    print("update stage %d H=%d: scale %s, gp max |err| / max |ref| %.2e" % (
        stage, H, sc, float((gp.double() - ref).abs().max() / ref.abs().max())))
    assert nbad == 0 and nsign == 0, "gp: %d elements outside the bound, %d signs differ" % (nbad, nsign)
    want = (p - torch.tensor(lr, dtype=torch.float32) * torch.sign(gp)).clamp(0.2, 0.7)
    assert torch.equal(p1, want), "sign step: %d elements differ" % int((p1 != want).sum())


# ---------------------------------------------------------------------------------------------------------------------
# K1^T
# ---------------------------------------------------------------------------------------------------------------------
LAUNCHES = {   # S -> launches (n0, n) over B = 2 images: the whole call, and one that starts in the middle of image 0
    1: [(0, 2), (1, 1)],
    5: [(0, 10), (2, 8)],
    129: [(0, 258), (1, 129)],       # 129 samples of image 0 (two passes of the 128-sample loop); 128 of 0 + 1 of 1
    300: [(0, 600), (44, 556)],      # 300 (three passes); 256 of image 0 added to G (two full passes) + 300 of image 1
}


def _occlusions(kind, H, N, rng):
    """(keep [N,H,H] bool on the device, hook arguments) for random rectangle tables or a random mask bank."""
    from dorpatch_b200 import masks as PM
    if kind == "rects":
        t = rng.randint(0, H + 1, (N, 4, 4))
        t[:, :, [0, 1]] = np.sort(t[:, :, [0, 1]], -1)
        t[:, :, [2, 3]] = np.sort(t[:, :, [2, 3]], -1)
        t[::5, 0, [0, 1]] = t[::5, 0, [1, 0]]                     # some empty
        t = np.ascontiguousarray(t, np.int16)
        keep = torch.from_numpy(~_occluded(t, H)).to(DEV)
        return keep, (t, C.c_void_p(t.ctypes.data), None, 0, None)
    M = 12
    occ = torch.from_numpy(rng.rand(M, H, H) < np.linspace(0.05, 0.9, M)[:, None, None])
    bank = PM.pack_bank(~occ, device=DEV)
    idx = np.ascontiguousarray(rng.randint(-1, M, (N, 2)), np.int32)
    occ = torch.cat([occ, torch.zeros(1, H, H, dtype=torch.bool)]).to(DEV)   # index -1: no mask
    keep = ~(occ[torch.from_numpy(idx[:, 0]).long()] | occ[torch.from_numpy(idx[:, 1]).long()])
    return keep, (idx, None, _ptr(bank), M, C.c_void_p(idx.ctypes.data), bank)


@_engines(["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("S", list(LAUNCHES))
def test_reduce_vs_fp64(eng, S):
    """K1^T (dp_debug_reduce) against the fp64 sum G[b] (+)= 2 sum_s keep_s dz_s over the launch's samples of image b,
    with dz [n,H,H,c_pad] drawn at the engine's dtype (NaN in the pad channels, which the kernel must not read).  An
    image whose first sample is in the launch is written (G filled with NaN first), any other added to (G holding
    random values); an image the launch does not touch stays NaN.  Per element |got - ref| <= 2 (n_s + 1) 2^-24
    (sum |2 dz| + |G before|).  Rectangles and a mask bank; pixel counts that are and are not multiples of 256."""
    precision, H = eng.precision, eng.img
    cp, dt = CPAD[precision], (torch.bfloat16 if precision == "bf16" else torch.float32)
    B, N = 2, 2 * S
    rng = np.random.RandomState(S * 1000 + H)
    gen = torch.Generator(device=DEV).manual_seed(S * 1000 + H)
    worst = 0.0
    for kind in ("rects", "bank"):
        keep, (hold, rp, bp, M, ip, *_bank) = _occlusions(kind, H, N, rng)
        for n0, n in LAUNCHES[S]:
            dz = torch.randn(n, H, H, cp, device=DEV, generator=gen).to(dt)
            dz[..., 3:] = float("nan")
            G0 = torch.randn(B, 3, H, H, device=DEV, generator=gen)
            G = torch.full((B, 3, H, H), float("nan"), device=DEV)
            added = []
            for b in range(B):
                lo, hi = max(n0, b * S), min(n0 + n, (b + 1) * S)
                if lo < hi and lo > b * S:
                    G[b] = G0[b]
                    added.append(b)
            _check(eng.lib.dp_debug_reduce(eng.handle, _ptr(dz), rp, bp, M, ip, B, S, n0, n, _ptr(G), eng._stream()))
            torch.cuda.synchronize()
            for b in range(B):
                lo, hi = max(n0, b * S), min(n0 + n, (b + 1) * S)
                if lo >= hi:
                    assert torch.isnan(G[b]).all(), "image %d outside the launch was written" % b
                    continue
                k = keep[lo:hi, :, :, None].double()
                d = dz[lo - n0:hi - n0, :, :, :3].double()
                ref = (2.0 * (k * d).sum(0)).permute(2, 0, 1)
                mag = (2.0 * (k * d.abs()).sum(0)).permute(2, 0, 1)
                if b in added:
                    ref, mag = ref + G0[b].double(), mag + G0[b].double().abs()
                err = (G[b].double() - ref).abs()
                bound = 2.0 * (hi - lo + 1) * 2.0 ** -24 * mag
                nbad = int((~(err <= bound)).sum())
                assert nbad == 0, "%s n0=%d n=%d image %d (%d samples, %s): %d elements outside the bound" % (
                    kind, n0, n, b, hi - lo, "added" if b in added else "written", nbad)
                worst = max(worst, float((err / bound.clamp_min(1e-30)).max()))
    print("reduce %s H=%d S=%d: worst error / bound %.3f" % (precision, H, S, worst))
