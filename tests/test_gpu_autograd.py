"""The differentiable native classifier (dp_eot_forward / dp_eot_backward, ops.eot_logits, the autograd path of
ResNetV2 / NormModel) against the engine's own fixed-loss paths (bit for bit) and against the oracle with torch
autograd (DESIGN §2 bars)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dorpatch_b200 import masks as PM
from oracle import attack as OA
from oracle import resnetv2 as OR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _rects(H, B, S, seed, dropout=2):
    table = PM.universe(H, dropout)
    idx = np.random.RandomState(seed).randint(0, table.shape[0], (B, S))
    return table, idx, PM.gather(table, idx)


def _cw_dlogits(logits, y, targeted, confidence, w):
    """d(w * sum_n cw_n)/d logits of the reference's CW loss (attack.py:16-23, its association order (confidence +
    other) - real; no top-2 ties in these inputs)."""
    N, K = logits.shape
    onehot = F.one_hot(y, K).bool()
    real = logits[torch.arange(N), y]
    oi = logits.masked_fill(onehot, float("-inf")).argmax(1)
    other = logits[torch.arange(N), oi]
    live = torch.where(targeted, (confidence + other) - real, (confidence + real) - other) >= 0
    d = torch.zeros_like(logits)
    sgn = torch.where(targeted, -1.0, 1.0).to(logits.device) * w
    d[torch.arange(N), y] = torch.where(live, sgn, 0.0)
    d[torch.arange(N), oi] = torch.where(live, -sgn, 0.0)
    return d


@pytest.fixture(scope="module")
def engines(oracle_params):
    """Engines of this module, freed at its end (the 224 px ones are large)."""
    from dorpatch_b200.engine import Engine
    made = {}

    def get(img, precision, chunk, max_images):
        key = (img, precision, chunk, max_images)
        if key not in made:
            e = Engine(img=img, precision=precision, chunk=chunk, max_images=max_images, autotune=False)
            e.load_state_dict(oracle_params)
            made[key] = e
        return made[key]
    yield get
    for e in made.values():
        e.close()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
def test_eot_forward_equals_predict(engines, precision):
    """dp_eot_forward's logits are dp_predict's, bit for bit: several chunks with a ragged last one, and plain
    classification (no rectangles)."""
    H, B, S = 112, 3, 5
    e = engines(H, precision, 4, 4)
    img = _rand((B, 3, H, H), 1).to(DEV)
    _, _, rects = _rects(H, B, S, 2)
    got = e.eot_forward(img, S, rects)
    _, ref = e.predict(img, S, rects, return_logits=True)
    assert np.array_equal(got.cpu().numpy(), ref)
    got1 = e.eot_forward(img, 1, None)
    _, ref1 = e.predict(img, 1, None, return_logits=True)
    assert np.array_equal(got1.cpu().numpy(), ref1)


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("B,S", [(1, 128), (4, 32)])
def test_eot_backward_of_cw_equals_attack_grad(engines, precision, B, S):
    """The CW gradient formed in torch from eot_forward's logits and pushed through eot_backward equals
    dp_attack_grad's grad_adv bit for bit (same kernels; dp_attack_grad adds only K4 and the regularisers)."""
    H = 224
    e = engines(H, precision, 64, 4)
    x, m, p = _rand((B, 3, H, H), 11).to(DEV), _rand((B, 1, H, H), 12).to(DEV), _rand((B, 3, H, H), 13).to(DEV)
    _, _, rects = _rects(H, B, S, 14)
    y = np.array([17, 400, 3, 999][:B])
    targeted = np.array([True, False, True, False][:B])
    G = torch.zeros(B, 3, H, H, device=DEV)
    r = e.attack_grad(x, m, p, rects, y, targeted, 0.1, 4.0, 1, G)
    adv, _, _ = e.paste(x, m, p, 4.0)
    logits = e.eot_forward(adv, S, rects)
    top2 = logits.topk(2, dim=1).values
    assert bool((top2[:, 0] > top2[:, 1]).all()), "inputs with a top-2 tie: pick other seeds"
    yy = torch.from_numpy(np.repeat(y, S)).to(DEV)
    tt = torch.from_numpy(np.repeat(targeted, S)).to(DEV)
    assert np.array_equal(logits.argmax(1).cpu().numpy(), r["preds"].reshape(-1))
    d = _cw_dlogits(logits, yy, tt, 0.1, 1.0 / S)
    g = e.eot_backward(d)
    torch.cuda.synchronize()
    assert torch.equal(g, G)


@pytest.mark.parametrize("H", [112, 224])
def test_cross_entropy_gradient_vs_oracle(engines, oracle_params, H):
    """fp32, cross-entropy over occluded samples: logits within 2e-3 of the oracle, input-gradient cosine >= 0.999
    against torch autograd on the oracle (DESIGN §2)."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    B, S = 2, 3
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    net.adopt_engine(engines(H, "fp32", 4, 4))
    img = _rand((B, 3, H, H), 21)
    table, idx, rects = _rects(H, B, S, 22)
    y = torch.tensor([5, 321]).repeat_interleave(S)
    xd = img.to(DEV).requires_grad_(True)
    logits = eot_logits(net, xd, rects, S)
    F.cross_entropy(logits, y.to(DEV)).backward()
    keep = torch.from_numpy(PM.to_bool(table, H)[idx])                      # [B,S,1,H,W]
    xr = img.clone().requires_grad_(True)
    ref = OR.forward(oracle_params, OA.occlude(xr[:, None], keep).reshape(B * S, 3, H, H))
    F.cross_entropy(ref, y).backward()
    err = (logits.detach().cpu() - ref.detach()).abs().max().item()
    cos = _cos(xd.grad.cpu(), xr.grad)
    print("H", H, "logit err", err, "grad cos", cos)
    assert err <= 2e-3
    assert cos >= 0.999


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_resident_and_recomputed_chunks_agree(engines, precision):
    """N = 3*chunk + 5 samples: the first chunks are recomputed in the backward, the last two are still resident.
    Whole images per chunk (chunk % S == 0): the gradient equals, bit for bit, the calls that each hold one chunk's
    images.  Images split across chunks (chunk % S != 0): it equals the sum, in chunk order, of the backwards of
    dlogits restricted to one chunk at a time.  A second backward of the same forward (other chunks resident) gives
    the same bits."""
    H = 112
    # whole images per chunk: chunk 4, S 1, 17 images
    e = engines(H, precision, 4, 17)
    B, S = 17, 1
    img = _rand((B, 3, H, H), 31).to(DEV)
    _, _, rects = _rects(H, B, S, 32)
    dl = (_rand((B * S, 1000), 33) - 0.5).to(DEV)
    e.eot_forward(img, S, rects)
    g = e.eot_backward(dl)
    g2 = e.eot_backward(dl)
    assert torch.equal(g, g2)
    parts = []
    for b0 in range(0, B, 4):
        e.eot_forward(img[b0:b0 + 4].contiguous(), S, rects[b0:b0 + 4])
        parts.append(e.eot_backward(dl[b0 * S:(b0 + 4) * S].contiguous()))
    assert torch.equal(g, torch.cat(parts))

    # images split across chunks: chunk 7, S 2, 13 images
    e = engines(H, precision, 7, 13)
    B, S = 13, 2
    img = _rand((B, 3, H, H), 34).to(DEV)
    _, _, rects = _rects(H, B, S, 35)
    dl = (_rand((B * S, 1000), 36) - 0.5).to(DEV)
    e.eot_forward(img, S, rects)
    g = e.eot_backward(dl)
    assert torch.equal(g, e.eot_backward(dl))
    acc = None
    for n0 in range(0, B * S, 7):
        d = torch.zeros_like(dl)
        d[n0:n0 + 7] = dl[n0:n0 + 7]
        gc = e.eot_backward(d)
        acc = gc if acc is None else acc + gc
    assert torch.equal(g, acc)


def _native_model(oracle_params, engine):
    """DataParallel(NormModel(ResNetV2)) on cuda:0 over an engine without timing trials, so that every call runs the
    same library algorithms (with several devices DataParallel would split the batch, and shards of another size run
    other algorithms)."""
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    net.adopt_engine(engine)
    return torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2")), device_ids=[0]).cuda().eval()


def test_module_autograd_semantics(engines, oracle_params):
    """DataParallel(NormModel(ResNetV2)) as a user drives it: model(x) with x.requires_grad and a loss's backward
    give eot_logits' gradient bit for bit; under no_grad the logits are those of the forward-only path; the weights get
    no gradient; double backward and a backward after another forward on the engine raise."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.utils import unwrap_native
    H, B = 112, 5                                          # two chunks of 4
    model = _native_model(oracle_params, engines(H, "fp32", 4, B))
    x0 = _rand((B, 3, H, H), 41).to(DEV)
    y = torch.tensor([1, 2, 3, 4, 5], device=DEV)

    x = x0.clone().requires_grad_(True)
    logits = model(x)
    F.cross_entropy(logits, y).backward()
    x2 = x0.clone().requires_grad_(True)
    logits2 = eot_logits(model, x2)
    F.cross_entropy(logits2, y).backward()
    assert torch.equal(logits, logits2)
    assert torch.equal(x.grad, x2.grad)
    assert all(p.grad is None for p in model.parameters())

    with torch.no_grad():
        l0 = model(x0)
    net = unwrap_native(model)
    _, ref = net.engine(H).predict(x0, 1, None, return_logits=True)
    assert np.array_equal(l0.cpu().numpy(), ref)
    assert torch.equal(l0, logits.detach())

    # the normalised-input module: same gradient through z = (x - 0.5) / 0.5 up to one rounding of the input
    z = ((x0 - 0.5) / 0.5).requires_grad_(True)
    F.cross_entropy(net(z), y).backward()
    assert _cos(z.grad, x.grad) >= 0.999

    x3 = x0.clone().requires_grad_(True)
    loss = F.cross_entropy(model(x3), y)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(loss, x3, create_graph=True)

    x4 = x0.clone().requires_grad_(True)
    loss = F.cross_entropy(model(x4), y)
    with torch.no_grad():
        model(x0)                                          # dp_predict on the same engine
    with pytest.raises(RuntimeError, match="stale forward"):
        loss.backward()
    assert x4.grad is None

    x5 = x0.clone().requires_grad_(True)
    loss = F.cross_entropy(model(x5), y)
    model(x0.clone().requires_grad_(True))                 # another differentiable forward
    with pytest.raises(RuntimeError, match="another eot_forward"):
        loss.backward()
    assert x5.grad is None


def test_user_written_sign_attack_matches_oracle(engines, oracle_params):
    """A targeted cross-entropy sign attack written in plain torch over eot_logits (20 steps, 16 occlusions per step,
    fp32, 112 px), and the same loop on the oracle.  At every step of the oracle's trajectory the native gradient at the
    same point agrees in sign with the oracle's on >= 99 % of the elements above 1e-3 of the largest, and the
    free-running native loop ends within 2 * iters * lr of the oracle's patch everywhere.  The fraction of patch pixels
    off is printed, not bounded: on this random-init classifier the loop is chaotic (a pixel moved by one step flips
    gradient signs elsewhere), so the two free-running trajectories drift apart on most pixels whatever the arithmetic."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, S, iters, lr, target = 112, 16, 20, 0.02, 123
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    net.adopt_engine(engines(H, "fp32", 8, 4))
    x = _rand((1, 3, H, H), 51)
    region = torch.zeros(1, 1, H, H)
    region[..., 30:70, 40:80] = 1.0
    table = PM.universe(H, 1)
    keep_all = torch.from_numpy(PM.to_bool(table, H))
    rs = np.random.RandomState(52)
    draws = [rs.randint(0, table.shape[0], (1, S)) for _ in range(iters)]
    yt = torch.full((S,), target)

    def grad(native, adv, idx):
        adv = adv.detach().requires_grad_(True)
        if native:
            loss = F.cross_entropy(eot_logits(net, adv, PM.gather(table, idx), S), yt.to(DEV))
        else:
            occ = OA.occlude(adv[:, None], keep_all[idx]).reshape(S, 3, H, H)
            loss = F.cross_entropy(OR.forward(oracle_params, occ), yt)
        loss.backward()
        return adv.grad

    def run(native, check=None):
        delta = torch.zeros(1, 3, H, H, device=DEV if native else "cpu")
        reg = region.to(delta.device)
        xx = x.to(delta.device)
        for idx in draws:
            adv = (xx + delta * reg).clamp(0, 1)
            g = grad(native, adv, idx) * reg
            if check is not None:
                check(adv, idx, g)
            delta = (delta - lr * g.sign()).clamp(-1, 1)
        return (delta * reg).cpu()

    agree = []

    def check(adv, idx, g_ref):
        g_nat = (grad(True, adv.to(DEV), idx) * region.to(DEV)).cpu()
        sure = g_ref.abs() > 1e-3 * g_ref.abs().max()
        agree.append((g_nat.sign() == g_ref.sign())[sure].float().mean().item())

    d_ref = run(False, check)
    d_nat = run(True)
    diff = (d_nat - d_ref).abs()
    off = (diff > 1e-6).float().sum().item() / region.sum().item() / 3
    print("per-step sign agreement min", min(agree), "pixels off", off, "max diff", diff.max().item())
    assert min(agree) >= 0.99
    assert diff.max().item() <= 2 * iters * lr + 1e-6
