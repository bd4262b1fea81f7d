"""Two-patch PatchCleanser window on the GPU: K1 on the 3- and 4-rectangle masks it needs (bit-exact), robust_predict
on the native engine against the oracle, and the main.py driver with --pc_n_patch 2."""
import contextlib
import io
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import two_patch as OT

pytestmark = pytest.mark.gpu
H = 112


def _slots(table):
    """[n,k,4] -> [n,4,4] int16, the k rectangles in slots 0..k-1, the rest empty."""
    out = np.zeros((len(table), 4, 4), np.int16)
    out[:, :table.shape[1]] = table
    return out


def _occlude_normalise_nhwc(img, rects):
    """numpy restatement of K1's non-fused output: (occlude(img, rects) - 0.5) / 0.5 as [n,H,W,3] float32, where
    occlude sets the union of each sample's <= 4 rectangles to 0.5 (PatchCleanser.py:99-100)."""
    z = ((img - np.float32(0.5)) / np.float32(0.5)).transpose(1, 2, 0)
    pos = np.arange(img.shape[-1])
    occ = np.zeros((len(rects), img.shape[-2], img.shape[-1]), bool)
    for s in range(4):
        r0, r1, c0, c1 = (rects[:, s, q].astype(np.int64)[:, None] for q in range(4))
        occ |= ((pos >= r0) & (pos < r1))[:, :, None] & ((pos >= c0) & (pos < c1))[:, None, :]
    return np.where(occ[..., None], np.float32(0.0), z[None])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_expand_three_and_four_rectangle_masks(engine_factory, precision):
    """K1 (dp_expand) over all 22 680 two-patch certificate masks of one ratio (3 rectangles each) and 300 second-round
    samples (two pairs, 4 rectangles, overlapping windows and repeated pairs included).  fp32: bit-exact; bf16: the bf16
    rounding of the fp32 result."""
    e = engine_factory(img=H, precision=precision, chunk=16, max_images=1)
    img = torch.rand(1, 3, H, H, generator=torch.Generator().manual_seed(11))
    cert = _slots(OT.rects_to_array(OT.mask_set_rects(H, 0.06, 2)))
    pairs = _slots(OT.rects_to_array(OT.mask_set_rects(H, 0.06, 1)))
    rng = np.random.RandomState(0)
    j, k = rng.randint(0, 630, 300), rng.randint(0, 630, 300)
    k[:10] = j[:10]
    round2 = pairs[j].copy()
    round2[:, 2:4] = pairs[k, 0:2]
    assert len(cert) == 22680 and cert[:, 2].any(axis=1).all() and round2[:, 3].any(axis=1).all()
    xd = img.cuda()
    for rects in [cert[i:i + 1260] for i in range(0, len(cert), 1260)] + [round2]:
        got = e.expand(xd, len(rects), rects).float().cpu()
        torch.cuda.synchronize()
        ref = torch.from_numpy(_occlude_normalise_nhwc(img[0].numpy(), rects))
        assert got.shape[-1] == e.c_pad and (got[..., 3:] == 0).all()
        if precision == "fp32":
            assert torch.equal(got[..., :3], ref)
        else:
            assert torch.equal(got[..., :3], ref.bfloat16().float())


@pytest.fixture(scope="module")
def native_model(oracle_params):
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    saved = {k: os.environ.get(k) for k in ("DORPATCH_PRECISION", "DORPATCH_CHUNK")}
    os.environ["DORPATCH_PRECISION"], os.environ["DORPATCH_CHUNK"] = "fp32", "64"
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    yield torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


# the oracle's round 1 on this image puts 4 of the 630 pairs off the majority (top-2 logit margins >= 0.007, far above
# fp32 noise), so the second round runs, and its CPU cost stays bounded (each disagreeing pair is 630 more forwards)
SEED, RATIO = 2, 0.015


def test_two_patch_patchcleanser_matches_oracle(native_model, oracle_net):
    """PatchCleanser(MaskWindow(112, r, 2)).robust_predict on the native fp32 engine vs the oracle: >= 97 % of the
    round-1 predictions and certificate bits agree, and where all of them do, prediction and certification are equal."""
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow, PatchCleanser
    img = torch.rand(3, H, H, generator=torch.Generator().manual_seed(SEED))
    pred, cert, p1, p2 = OT.robust_predict(oracle_net, img, H, RATIO, certify=True)
    labels, counts = torch.from_numpy(p1).unique(sorted=False, return_counts=True)
    assert 1 <= int((p1 != labels[counts.argmax()].item()).sum()) <= 4
    with contextlib.redirect_stdout(io.StringIO()):
        rec = PatchCleanser(MaskWindow(H, RATIO, 2), native_model).robust_predict(img.cuda(), True)
    assert rec.preds_1.shape == (630,) and np.asarray(rec.preds_2).shape == (22680,) and p2.shape == (22680,)
    b1, b2 = rec.preds_1 == p1, np.asarray(rec.preds_2).astype(bool) == p2.astype(bool)
    print("round 1 agreement %.4f, certificate agreement %.4f" % (b1.mean(), b2.mean()))
    assert b1.mean() >= 0.97 and b2.mean() >= 0.97
    if b1.all() and b2.all():
        assert rec.prediction == pred and bool(rec.certification) == bool(cert)


def test_main_driver_two_patch(tmp_path, monkeypatch):
    """main.py --pc_n_patch 2: two-patch records in adv_PC2_<i>.pt, the usual metrics line; a second run reuses the
    patches and the records; a default run on the same directory then adds the one-patch adv_PC_<i>.pt."""
    from dorpatch_b200 import main as M
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("DORPATCH_PRECISION", "bf16")
    monkeypatch.setenv("DORPATCH_CHUNK", "128")
    base = ["--synthetic", "2", "--random_init", "--img_size", str(H), "--max_iterations", "3", "--sampling_size", "4",
            "--dropout", "1", "--num_batches", "2", "--chunk", "128"]

    def run(extra):
        with contextlib.redirect_stdout(io.StringIO()):
            return M.cli(base + extra)

    def records(name):
        with open(os.path.join(rd, name), "rb") as f:
            return pickle.load(f)

    out = run(["--pc_n_patch", "2"])
    rd = out["result_dir"]
    assert rd.endswith("num_patch=-1_patch_budget=0.12")                # --pc_n_patch is not part of the path
    assert out["line"].startswith("clean accuracy: ") and "certified_ASR@PC:" in out["line"] and len(out["acc_PC"]) == 4
    stored = ["adv_mask_%d.pt" % i for i in range(2)] + ["adv_pattern_%d.pt" % i for i in range(2)] + \
             ["adv_PC2_%d.pt" % i for i in range(2)]
    for f in stored:
        assert os.path.exists(os.path.join(rd, f)), f
    assert not any(os.path.exists(os.path.join(rd, "adv_PC_%d.pt" % i)) for i in range(2))
    recs = records("adv_PC2_0.pt")
    assert len(recs[0]) == 4
    assert all(r.preds_1.shape == (630,) and np.asarray(r.preds_2).shape == (22680,) for r in recs[0])
    mtimes = {f: os.stat(os.path.join(rd, f)).st_mtime_ns for f in stored}

    again = run(["--pc_n_patch", "2"])
    assert again["result_dir"] == rd and again["line"] == out["line"]
    assert {f: os.stat(os.path.join(rd, f)).st_mtime_ns for f in stored} == mtimes

    one = run([])
    assert one["result_dir"] == rd
    assert {f: os.stat(os.path.join(rd, f)).st_mtime_ns for f in stored} == mtimes
    recs = records("adv_PC_0.pt")
    assert len(recs[0]) == 4 and recs[0][0].preds_1.shape == (36,) and recs[0][0].preds_2.shape == (630,)
