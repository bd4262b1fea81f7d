"""Mask banks (arbitrary occlusion masks) through every kernel that reads them: K1 bit for bit against numpy at every
input layout, the bank against the rectangle path on the same occlusions (logits and gradients bit for bit), masks that
are not rectangles against the oracle with torch autograd, the fused bf16 stem backward against torch, PatchCleanser
with a window given only as bool mask sets, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dorpatch_b200 import masks as PM
from oracle import attack as OA
from oracle import resnetv2 as OR
from test_gpu_occlusion import LAYOUTS, _degenerate_table, _engine, _occluded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _shapes(H, n_random=8, seed=0):
    """[n,H,H] bool occluded sets that are not (all) rectangles: discs, a checkerboard, single pixels, the full image,
    the last column, single rows on row-tile borders, a ring, a diagonal, random noise."""
    yy, xx = np.mgrid[0:H, 0:H]
    occ = [
        (yy - H * 0.4) ** 2 + (xx - H * 0.6) ** 2 < (H * 0.2) ** 2,
        (yy - 3) ** 2 + (xx - (H - 2)) ** 2 < 36,                    # a disc cut by two edges
        ((yy // 3) + (xx // 5)) % 2 == 0,                            # checkerboard
        (yy == 17) & (xx == 23),
        (yy == H - 1) & (xx == H - 1),
        np.ones((H, H), bool),
        xx == H - 1,
        (yy == 7) | (yy == 8) | (yy == 15) | (yy == 16),
        np.abs(np.hypot(yy - H / 2, xx - H / 2) - H / 4) < 2,
        np.abs(yy - xx) <= 1,
        np.zeros((H, H), bool),
    ]
    rng = np.random.RandomState(seed)
    occ += list(rng.rand(n_random, H, H) < 0.2)
    return np.stack(occ)


def _bank(occ):
    return PM.pack_bank(torch.from_numpy(~occ), device=DEV)


def _sample_occlusions(H, seed):
    """Occluded sets [n,H,H] and the bank index pairs that select them: every shape alone, then pairs of shapes and
    pairs with one slot empty."""
    occ = _shapes(H, seed=seed)
    n = len(occ)
    rng = np.random.RandomState(seed + 1)
    pairs = np.stack([rng.randint(0, n, 12), rng.randint(-1, n, 12)], 1)
    pairs[0] = (-1, -1)
    pairs[1] = (-1, 3)
    idx = np.concatenate([np.stack([np.arange(n), np.full(n, -1)], 1), pairs]).astype(np.int32)
    sel = np.zeros((len(idx), H, H), bool)
    for k, (a, b) in enumerate(idx):
        if a >= 0:
            sel[k] |= occ[a]
        if b >= 0:
            sel[k] |= occ[b]
    return occ, idx, sel


def _normalised(img, occluded):
    z = ((img - np.float32(0.5)) / np.float32(0.5)).transpose(1, 2, 0)
    return np.where(occluded[..., None], np.float32(0.0), z[None])


@pytest.mark.parametrize("precision,env,cp", LAYOUTS, ids=["bf16-c3", "bf16-c8", "bf16-c4", "fp32-c4", "fp32-c8"])
def test_expand_bank_bit_exact(oracle_params, precision, env, cp):
    """K1 (dp_expand_bank) bit for bit against numpy: the degenerate rectangle tables rasterised into a bank, and
    masks that are not rectangles with one or two indices per sample; three launch shapes and both store modes."""
    H = 112
    e = _engine(oracle_params, precision, **env)
    try:
        assert e.c_pad == cp
        rects = _degenerate_table(H)
        occ_r = _occluded(rects, H)
        occ, idx, sel = _sample_occlusions(H, 3)
        bank = _bank(np.concatenate([occ_r, occ]))
        idx_all = np.concatenate([np.stack([np.arange(len(rects)), np.full(len(rects), -1)], 1),
                                  np.where(idx >= 0, idx + len(rects), -1)]).astype(np.int32)
        want = np.concatenate([occ_r, sel])
        img = _rand((1, 3, H, H), 5)
        ref = torch.from_numpy(_normalised(img[0].numpy(), want))
        if precision == "bf16":
            ref = ref.bfloat16().float()
        for rows, sg, mode in ((0, 0, 0), (0, 1, 0), (0, 0, 1), (4, 2, 0)):
            e.lib.dp_debug_k1_tuning(rows, sg, mode)
            got = e.expand_bank(img.to(DEV), len(idx_all), bank, idx_all).float().cpu()
            torch.cuda.synchronize()
            assert got.shape == (len(idx_all), H, H, cp) and (got[..., 3:] == 0).all()
            bad = (got[..., :3] != ref).any(-1).any(-1).any(-1).nonzero().flatten().tolist()
            assert not bad, ("launch shape", rows, sg, mode, "samples", bad[:8])
            if mode == 0 and rows == 0 and sg == 0:                # equals the rectangle path on the rectangles
                gr = e.expand(img.to(DEV), len(rects), rects).float().cpu()
                assert torch.equal(gr, got[:len(rects)])
    finally:
        e.lib.dp_debug_k1_tuning(0, 0, 0)
        e.close()


def _dual_case(H, B, S, seed):
    """Rectangle tables that occlude like a bank selection: each sample is the union of two single window masks, as
    rects (slots 0-1 and 2-3, masks.gather with idx_dual) and as bank index pairs."""
    table = PM.universe(H, 1)                                      # [144,2,4] single masks
    rng = np.random.RandomState(seed)
    a, b = rng.randint(0, len(table), (B, S)), rng.randint(0, len(table), (B, S))
    b[:, 0] = -1                                                   # some samples with one mask only
    rects = PM.gather(table, a, idx_dual=np.where(b >= 0, b, 0))
    rects[:, 0, 2:4] = 0
    bank = PM.pack_bank(PM.to_bool(table, H), device=DEV)
    return rects, bank, np.stack([a, b], -1)


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16", "bf16-pool"])
def test_bank_equals_rectangles(oracle_params, precision):
    """The same occlusions as rectangles and as a bank: predict and eot_forward logits and the eot_logits input gradient
    (K1^T at fp32 / tf32, the fused stem backward at bf16, with the max-pool backward fused in as well) are bit for bit
    the rectangle path's; images straddle chunks and the first chunks are recomputed in the backward."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, B, S = 112, 3, 7
    env = {"DORPATCH_POOL_BWD": "fused"} if precision == "bf16-pool" else {}
    e = _engine(oracle_params, precision.split("-")[0], chunk=4, max_images=B, **env)
    try:
        rects, bank, idx = _dual_case(H, B, S, 7)
        img = _rand((B, 3, H, H), 8).to(DEV)
        pr, lr = e.predict(img, S, rects, return_logits=True)
        pb, lb = e.predict(img, S, bank=bank, idx=idx.reshape(-1, 2), return_logits=True)
        assert np.array_equal(lr, lb) and np.array_equal(pr, pb)
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        y = torch.from_numpy(np.arange(B * S) * 37 % 1000).to(DEV)
        grads, logits = [], []
        for kw in (dict(rects=rects), dict(bank=bank, idx=idx)):
            x = img.clone().requires_grad_(True)
            out = eot_logits(net, x, S=S, **kw)
            F.cross_entropy(out, y).backward()
            grads.append(x.grad)
            logits.append(out.detach())
        torch.cuda.synchronize()
        assert torch.equal(logits[0], logits[1]) and np.array_equal(logits[1].cpu().numpy(), lb)
        assert torch.equal(grads[0], grads[1]) and grads[0].abs().sum() > 0
    finally:
        e.close()


def test_param_grads_bank_equals_rectangles(oracle_params):
    """param_grads=True through a bank-occluded forward: parameter gradients bit for bit the rectangle path's."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, B, S = 112, 2, 5
    e = _engine(oracle_params, "fp32", chunk=4, max_images=B)
    try:
        rects, bank, idx = _dual_case(H, B, S, 9)
        img = _rand((B, 3, H, H), 10).to(DEV)
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        for k, p in net.named_parameters():
            p.requires_grad_(k.startswith("stem") or k.startswith("head") or k.startswith("stages.3"))
        y = torch.from_numpy(np.arange(B * S) * 11 % 1000).to(DEV)
        got = []
        for kw in (dict(rects=rects), dict(bank=bank, idx=idx)):
            net.zero_grad(set_to_none=True)
            x = img.clone().requires_grad_(True)
            F.cross_entropy(eot_logits(net, x, S=S, param_grads=True, **kw), y).backward()
            got.append([x.grad] + [p.grad.clone() for _, p in net.named_parameters() if p.requires_grad])
        torch.cuda.synchronize()
        assert len(got[0]) > 2
        for a, b in zip(*got):
            assert torch.equal(a, b)
    finally:
        e.close()


@pytest.mark.parametrize("H", [112, 224])
def test_non_rectangular_masks_vs_oracle(oracle_params, H):
    """fp32, cross-entropy over samples occluded by masks that are not rectangles (discs, a ring, a diagonal band, a
    checkerboard, single pixels and rows, one or two per sample): logits within 2e-3 of the oracle and input-gradient
    cosine >= 0.999 against torch autograd on the oracle (the bars of test_gpu_autograd.py).  Chunk 4 with 2 x 5
    samples: the backward recomputes the first chunk, and a second backward gives the same bits.  A fully occluded
    sample is left out: its input is constant, every GroupNorm then normalises a (nearly) constant tensor, and the
    classifier's logits differ from the oracle's by 8e-3 whichever occlusion format produced it (K1 writes it bit for
    bit, test_expand_bank_bit_exact); every other sample is within 6e-6."""
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    B, S = 2, 5
    e = _engine(oracle_params, "fp32", img=H, chunk=4, max_images=B)
    try:
        occ = _shapes(H, n_random=0)
        bank = _bank(occ)
        partial = np.array([i for i in range(len(occ)) if not occ[i].all()])
        rng = np.random.RandomState(12)
        idx = np.stack([partial[rng.randint(0, len(partial), (B, S))], rng.choice(np.append(partial, -1), (B, S))], -1)
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        img = _rand((B, 3, H, H), 13)
        y = torch.tensor([5, 321]).repeat_interleave(S)
        xd = img.to(DEV).requires_grad_(True)
        logits = eot_logits(net, xd, S=S, bank=bank, idx=idx)
        F.cross_entropy(logits, y.to(DEV)).backward(retain_graph=True)
        g1 = xd.grad.clone()
        xd.grad = None
        F.cross_entropy(logits, y.to(DEV)).backward()
        assert torch.equal(g1, xd.grad)
        o = occ[idx[..., 0]] | np.where(idx[..., 1:2, None] >= 0, occ[np.maximum(idx[..., 1], 0)], False)
        keep = torch.from_numpy(~o)[:, :, None]                      # [B,S,1,H,W]
        xr = img.clone().requires_grad_(True)
        ref = OR.forward(oracle_params, OA.occlude(xr[:, None], keep).reshape(B * S, 3, H, H))
        F.cross_entropy(ref, y).backward()
        per = (logits.detach().cpu() - ref.detach()).abs().amax(1)
        scale = ref.detach().abs().amax(1)
        cos = _cos(g1.cpu(), xr.grad)
        print("H", H, "logit err per sample", per.tolist(), "max |logit|", scale.tolist(), "grad cos", cos)
        assert float(per.max()) <= 2e-3 and cos >= 0.999
    finally:
        e.close()


def test_bf16_stem_bwd_reduce_bank_vs_torch(oracle_params):
    """The fused stem dgrad + masked reduce reading a bank against torch fp32 conv_transpose2d on the same bf16
    operands, at the bounds of test_gpu_occlusion.py; two images, the second starting mid-launch."""
    from dorpatch_b200 import _lib
    H = 112
    e = _engine(oracle_params, "bf16")
    try:
        occ, idx, sel = _sample_occlusions(H, 14)
        bank = _bank(occ)
        N = len(idx) - len(idx) % 2
        B, S = 2, N // 2
        idx, sel = np.ascontiguousarray(idx[:N]), sel[:N]
        hs = H // 2
        dY = (_rand((N, hs, hs, 64), 15) * 2e-2 - 1e-2).to(torch.bfloat16)
        G = torch.empty(B, 3, H, H, device=DEV)
        dYd = dY.to(DEV)
        _lib.check(e.lib.dp_debug_stem_bwd_reduce_bank(e.handle, C.c_void_p(dYd.data_ptr()), C.c_void_p(bank.data_ptr()),
                                                       len(occ), C.c_void_p(idx.ctypes.data), B, S,
                                                       C.c_void_p(G.data_ptr()), e._stream()))
        torch.cuda.synchronize()
    finally:
        e.close()
    w = OR.standardize(oracle_params["stem.conv.weight"]).to(torch.bfloat16).float()
    dX = F.conv_transpose2d(dY.float().permute(0, 3, 1, 2), w, stride=2, padding=3, output_padding=1)
    ref = 2.0 * (dX * torch.from_numpy(~sel).float()[:, None]).reshape(B, S, 3, H, H).sum(1)
    got = G.cpu()
    rel = float((got - ref).norm() / ref.norm())
    mx = float((got - ref).abs().max() / ref.abs().max())
    print("stem_bwd_reduce, bank: rel L2 %.2e, max abs / max %.2e" % (rel, mx))
    assert rel <= 1e-5 and mx <= 1e-4, (rel, mx)


class _BoolWindow:
    """A PatchCleanser window that is only its bool mask sets (what the reference's PatchCleanser reads)."""

    def __init__(self, single, double):
        self.mask_set, self.double_mask_set = single, double


def _second_round_images(pc, H, n, seeds):
    """Candidate images (uniform noise with a high-contrast square; seed -1: flat grey, which every occlusion leaves
    unchanged, so its first round is unanimous) split by whether the bank path's first round is unanimous:
    (unanimous seeds, second-round seeds)."""
    singles = pc._bank("mask_set", torch.empty(0, device=DEV))
    one, two = [], []
    for seed in seeds:
        img = _patch_image(H, seed)
        p1 = pc._predict_bank(img, singles, np.arange(n))
        (two if len(np.unique(p1)) > 1 else one).append(seed)
    return one, two


def _patch_image(H, seed):
    if seed < 0:                                                   # flat grey: every occlusion leaves it unchanged
        return torch.full((3, H, H), 0.5, device=DEV)
    img = _rand((3, H, H), seed).to(DEV)
    r0, c0 = (seed * 7) % (H // 2), (seed * 13) % (H // 2)
    sq = img[:, r0:r0 + H // 4, c0:c0 + H // 4]
    img[:, r0:r0 + H // 4, c0:c0 + H // 4] = 0.5 + 0.5 * torch.sign(sq - 0.5)   # a high-contrast patch
    return img


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("n_patch", [1, 2])
def test_patchcleanser_bool_window_equals_mask_window(oracle_params, precision, n_patch):
    """A duck-typed window holding MaskWindow's bool sets gives MaskWindow's records (prediction, certification,
    preds_1, preds_2) through the bank path, on an image whose first round is unanimous and on one that takes the
    second round (both are asserted to be among the candidates; the unanimous one is the first found, flat grey at
    the latest)."""
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow, PatchCleanser
    from dorpatch_b200.resnetv2 import ResNetV2
    H = 112
    e = _engine(oracle_params, precision, chunk=64, max_images=1)
    try:
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        mw = MaskWindow(H, 0.06 if n_patch == 1 else 0.03, n_patch)
        bw = _BoolWindow(mw.mask_set, mw.double_mask_set)
        pa, pb = PatchCleanser(mw, net), PatchCleanser(bw, net)
        one, two = _second_round_images(pb, H, len(mw.mask_rects), [-1] + list(range(16, 48)))
        assert one and two, (one, two)
        for seed in (one[0], two[0]):
            img = _patch_image(H, seed)
            ra, rb = pa.robust_predict(img, certify=True), pb.robust_predict(img, certify=True)
            assert ra.prediction == rb.prediction and ra.certification == rb.certification
            assert np.array_equal(ra.preds_1, rb.preds_1) and np.array_equal(ra.preds_2, rb.preds_2)
        assert len(np.unique(rb.preds_1)) > 1
    finally:
        e.close()


def _oracle_model(oracle_params):
    def model(x):
        with torch.no_grad():
            return OR.forward(oracle_params, x.cpu().float())
    return model


def test_patchcleanser_non_rectangular_window_vs_oracle(oracle_params, monkeypatch):
    """fp32, 56 px, a window of disc / ring occluders (not rectangles): records equal to the oracle's robust_predict
    (oracle/patchcleanser.py) run on the same bool sets, on an image whose first round is unanimous and on one that
    takes the second round."""
    from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
    from dorpatch_b200.resnetv2 import ResNetV2
    from test_mask_bank_patchcleanser import _custom_sets, _oracle_records
    H = 56
    single, double = _custom_sets(H)
    e = _engine(oracle_params, "fp32", img=H, chunk=64, max_images=1)
    try:
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        pc = PatchCleanser(_BoolWindow(single, double), net)
        one, two = _second_round_images(pc, H, len(single), range(50, 82))
        assert one and two, (one, two)
        for seed in (one[0], two[0]):
            img = _patch_image(H, seed)
            got = pc.robust_predict(img, certify=True)
            pred, cert, p1, p2 = _oracle_records(_oracle_model(oracle_params), img.cpu(), single, double, monkeypatch)
            assert got.prediction == pred and got.certification == cert
            assert np.array_equal(got.preds_1, p1) and np.array_equal(got.preds_2, p2)
        assert len(np.unique(p1)) > 1
    finally:
        e.close()


@pytest.mark.parametrize("targeted", [False, True])
def test_collect_failure_non_rectangular_universe_vs_oracle(oracle_params, targeted):
    """fp32, 56 px: collect_failure on a bool universe that from_bool cannot decompose (it takes the bank path) returns
    the failed indices of the oracle's collect_failure (oracle/attack.py) over the same universe, images united."""
    from dorpatch_b200.attack import DorPatch
    from dorpatch_b200.resnetv2 import ResNetV2
    from oracle import attack as OAt
    H, B = 56, 2
    e = _engine(oracle_params, "fp32", img=H, chunk=16, max_images=B)
    try:
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        occ = _shapes(H, n_random=4, seed=18)
        universe = torch.from_numpy(~occ)[:, None]
        with pytest.raises(NotImplementedError):
            PM.from_bool(universe)
        img = torch.stack([_patch_image(H, 19), _patch_image(H, 20)])
        model = _oracle_model(oracle_params)
        y = model(img).argmax(1)                                   # the clean predictions
        got = DorPatch().collect_failure(img, y, universe, targeted, net)
        want = set()
        for b in range(B):
            want |= set(OAt.collect_failure(model, img[b:b + 1].cpu(), y[b], universe, targeted, 8))
        assert got == sorted(want), (got, sorted(want))
        if not targeted:
            assert 10 in got                                       # the empty mask keeps every clean prediction
    finally:
        e.close()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_bank_resident_and_recomputed_chunks_agree(oracle_params, precision):
    """Bank occlusion, whole images per chunk (chunk 4, S 2, 6 images): the backward of one call, whose first chunk
    the engine recomputes, equals bit for bit the calls that each hold their single chunk resident."""
    H, B, S = 112, 6, 2
    e = _engine(oracle_params, precision, chunk=4, max_images=B)
    try:
        occ = _shapes(H, n_random=2, seed=21)
        bank = _bank(occ)
        rng = np.random.RandomState(22)
        idx = np.stack([rng.randint(0, len(occ), (B, S)), rng.randint(-1, len(occ), (B, S))], -1).astype(np.int32)
        img = _rand((B, 3, H, H), 23).to(DEV)
        dl = (_rand((B * S, 1000), 24) - 0.5).to(DEV)
        e.eot_forward(img, S, bank=bank, idx=idx.reshape(-1, 2))
        g = e.eot_backward(dl)
        parts = []
        for b0 in range(0, B, 2):
            e.eot_forward(img[b0:b0 + 2].contiguous(), S, bank=bank, idx=idx[b0:b0 + 2].reshape(-1, 2))
            parts.append(e.eot_backward(dl[b0 * S:(b0 + 2) * S].contiguous()))
        torch.cuda.synchronize()
        assert torch.equal(g, torch.cat(parts)) and g.abs().sum() > 0
    finally:
        e.close()


def test_bank_refusals(oracle_params):
    """A bank with rects or xforms, indices outside [-1, n_bank), a null bank with an index, n_bank < 1, and a bank
    changed in place before the backward are refused."""
    from dorpatch_b200 import _lib
    from dorpatch_b200.ops import eot_logits
    from dorpatch_b200.resnetv2 import ResNetV2
    H, B, S = 112, 1, 2
    e = _engine(oracle_params, "fp32", chunk=4, max_images=B)
    try:
        occ = _shapes(H, n_random=0)
        bank = _bank(occ)
        img = _rand((B, 3, H, H), 20).to(DEV)
        idx = np.array([[0, 1], [2, -1]], np.int32)
        with pytest.raises(ValueError):
            e.predict(img, S, np.zeros((B, S, 4, 4), np.int16), bank=bank, idx=idx)
        with pytest.raises(ValueError):
            e.eot_forward(img, S, xforms=np.zeros((B, S, 8), np.float32), bank=bank, idx=idx)
        for bad in (np.array([[0, len(occ)], [0, 0]], np.int32), np.array([[-2, 0], [0, 0]], np.int32)):
            with pytest.raises(ValueError):
                e.predict(img, S, bank=bank, idx=bad)
        logits = torch.empty(B * S, 1000, device=DEV)
        ok = np.ascontiguousarray(idx)
        for bp, nb, ix in ((C.c_void_p(bank.data_ptr()), len(occ), np.array([[0, len(occ)], [0, 0]], np.int32)),
                           (None, len(occ), ok), (C.c_void_p(bank.data_ptr()), 0, np.full((2, 2), -1, np.int32))):
            rc = e.lib.dp_eot_forward_bank(e.handle, C.c_void_p(img.data_ptr()), B, S, bp, nb, C.c_void_p(ix.ctypes.data),
                                           C.c_void_p(logits.data_ptr()), e._stream())
            assert rc != 0 and b"dp_eot_forward_bank" in e.lib.dp_last_error()
        net = ResNetV2(seed=0)
        net.load_state_dict(oracle_params)
        net.adopt_engine(e)
        x = img.clone().requires_grad_(True)
        out = eot_logits(net, x, S=S, bank=bank, idx=idx.reshape(B, S, 2))
        bank.add_(0)                                                    # an in-place change (same values)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            out.sum().backward()
        e.eot_forward(img, S, bank=bank, idx=idx)
        bank.add_(0)
        with pytest.raises(RuntimeError, match="mask bank"):
            e.eot_backward(torch.ones(B * S, 1000, device=DEV))
    finally:
        e.close()
