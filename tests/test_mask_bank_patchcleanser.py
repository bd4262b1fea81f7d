"""PatchCleanser on a window given only as bool mask sets (the mask-bank path) on the CPU, with the classifier replaced
by TinyNet: its records and its calls equal the rectangle path's on MaskWindow's own sets, including the second round's
(mask j, mask k) pairs, and a window of masks that are not rectangles gives the records of the oracle's
robust_predict (oracle/patchcleanser.py) run on the same bool sets.  Bit-exact throughout; no GPU needed."""
import contextlib
import importlib.util
import io
import os
import types

import numpy as np
import pytest
import torch

from dorpatch_b200 import masks as PM
from oracle import patchcleanser as OPC

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, "golden", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MG = _load("make_two_patch_golden")
TINY = _load("make_golden").TinyNet().eval()


def _tiny_preds(x):
    with torch.no_grad():
        return TINY(x).argmax(1)


class _BoolWindow:
    """A window that is only its bool mask sets, as the reference's PatchCleanser reads them."""

    def __init__(self, single, double):
        self.mask_set, self.double_mask_set = single, double


class _TinyBankPatchCleanser:
    """PatchCleanser on a bool-set window with the engine replaced by TinyNet: each sample is the image occluded by
    the masks its index pair selects from the bank, unpacked -- so the bank packing, the pair construction of the second
    round and the control flow are what the tests check."""

    def __init__(self, window):
        from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
        from dorpatch_b200.resnetv2 import ResNetV2
        self.calls = []
        self.pc = PatchCleanser(window, ResNetV2())
        self.pc._predict_bank = self._predict_bank

    def _predict_bank(self, img, bank, idx):
        idx = np.asarray(idx)
        if idx.ndim == 1:                                          # one mask per sample
            idx = np.stack([idx, np.full(len(idx), -1)], 1)
        self.calls.append(idx.copy())
        keep = PM.unpack_bank(bank, img.shape[-1])                  # [M,1,H,W]
        k = torch.ones((len(idx),) + keep.shape[1:], dtype=torch.bool)
        for c in range(idx.shape[1]):
            sel = torch.from_numpy(idx[:, c].astype(np.int64))
            k &= torch.where((sel >= 0)[:, None, None, None], keep[sel.clamp(min=0)], torch.ones_like(k))
        return _tiny_preds(img * k + 0.5 * ~k).numpy().astype(np.int32)


class _TinyRectPatchCleanser:
    """The rectangle path (MaskWindow's tables) with the same TinyNet classifier."""

    def __init__(self, mw):
        from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
        from dorpatch_b200.resnetv2 import ResNetV2
        self.pc = PatchCleanser(mw, ResNetV2())
        self.pc._predict = self._predict

    def _predict(self, img, rects):
        keep = torch.from_numpy(PM.to_bool(rects, img.shape[-1]))
        return _tiny_preds(img * keep + 0.5 * ~keep).numpy().astype(np.int32)


def _records_equal(a, b):
    return (a.prediction == b.prediction and a.certification == b.certification and np.array_equal(a.preds_1, b.preds_1)
            and np.array_equal(a.preds_2, b.preds_2))


def _mask_window(H, r, n_patch):
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow
    with contextlib.redirect_stdout(io.StringIO()):
        return MaskWindow(H, r, n_patch)


@pytest.mark.parametrize("seed", MG.SEEDS)
def test_bool_window_equals_mask_window(seed):
    """MaskWindow(56, 0.12) and a window holding only its bool sets give the same records; the second round asks for
    every single j paired with each disagreeing single k, and the certificate for the doubles in order."""
    mw = _mask_window(56, 0.12, 1)
    img = MG.two_patch_image(seed)
    ref = _TinyRectPatchCleanser(mw).pc.robust_predict(img, True)
    t = _TinyBankPatchCleanser(_BoolWindow(mw.mask_set, mw.double_mask_set))
    got = t.pc.robust_predict(img, True)
    assert _records_equal(ref, got)
    labels, counts = torch.from_numpy(got.preds_1).unique(sorted=False, return_counts=True)
    majority = labels[counts.argmax()].item()
    want = [np.stack([np.arange(36), np.full(36, -1)], 1)]
    for label in labels.tolist():
        if label != majority:
            for k in np.nonzero(got.preds_1 == label)[0]:
                want.append(np.stack([np.arange(36), np.full(36, k)], 1))
    want.append(np.stack([np.arange(630), np.full(630, -1)], 1))
    assert len(t.calls) == len(want)
    for c, w in zip(t.calls, want):
        assert np.array_equal(c, w)
    if seed == 1158:
        assert len(labels) > 1                                     # this image takes the second round


def _custom_sets(H):
    """36 disc / ring occluders on a 6 x 6 grid and 48 unions of two of them -- none a union of <= 2 rectangles."""
    yy, xx = np.mgrid[0:H, 0:H]
    c = (np.arange(6) + 0.5) * H / 6
    occ = []
    for i in range(6):
        for j in range(6):
            d = np.hypot(yy - c[i], xx - c[j])
            occ.append(d < H / 5 if (i + j) % 2 == 0 else np.abs(d - H / 7) < H / 14)
    occ = np.stack(occ)
    rng = np.random.RandomState(0)
    pairs = rng.randint(0, 36, (48, 2))
    double = occ[pairs[:, 0]] | occ[pairs[:, 1]]
    return ~occ[:, None], ~double[:, None]


def _oracle_records(model, img, single, double, monkeypatch):
    """oracle.patchcleanser.robust_predict on the given bool sets: its mask sets come from oracle.masks, which is
    swapped here for one that returns these sets."""
    stub = types.SimpleNamespace(mask_set_rects=lambda H, r, dropout: dropout,
                                 rects_to_bool=lambda dropout, H: single if dropout == 1 else double)
    with monkeypatch.context() as m:
        m.setattr(OPC, "omasks", stub)
        return OPC.robust_predict(model, img, img.shape[-1], 0.0, certify=True)


def test_non_rectangular_window_matches_oracle(monkeypatch):
    """A window of disc / ring occluders: records equal to the oracle's on the same bool sets, with TinyNet as the
    classifier, on images that take the unanimous branch and the second round."""
    single, double = _custom_sets(56)
    with pytest.raises(NotImplementedError):
        PM.from_bool(single)
    rounds = set()
    for seed in MG.SEEDS:
        img = MG.two_patch_image(seed)
        got = _TinyBankPatchCleanser(_BoolWindow(single, double)).pc.robust_predict(img, True)
        pred, cert, p1, p2 = _oracle_records(TINY, img, single, double, monkeypatch)
        assert got.prediction == pred and got.certification == cert
        assert np.array_equal(got.preds_1, p1) and np.array_equal(got.preds_2, p2)
        rounds.add(len(np.unique(p1)) > 1)
    assert rounds == {False, True}, rounds
