"""Two-patch PatchCleanser window (MaskWindow(img, r, n_patch=2)) on the CPU: the oracle pinned to the fixture the
unmodified reference produced (tests/golden/make_two_patch_golden.py), the product's rectangle tables equal to the
oracle's, and PatchCleanser.robust_predict's control flow over those tables equal to the reference's records.
Bit-exact throughout; no GPU needed."""
import contextlib
import importlib.util
import io
import os

import numpy as np
import pytest
import torch

from dorpatch_b200 import masks as PM
from oracle import masks as OM
from oracle import two_patch as OT

HERE = os.path.dirname(os.path.abspath(__file__))
RATIOS = (0.015, 0.03, 0.06, 0.12)


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, "golden", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MG = _load("make_two_patch_golden")
G = MG.load()


def _tiny():
    return _load("make_golden").TinyNet().eval()


def _mask_window(H, r, n_patch):
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow
    with contextlib.redirect_stdout(io.StringIO()):
        return MaskWindow(H, r, n_patch)


@pytest.mark.parametrize("H", [56, 224])
@pytest.mark.parametrize("r", RATIOS)
def test_oracle_two_patch_geometry_matches_reference(H, r):
    assert tuple(G["tp_geom_%d_%s" % (H, r)]) == OT.window_geometry(H, r)
    pairs = OT.mask_set_rects(H, r, 1)
    assert len(pairs) == 630
    if H == 56:
        assert np.array_equal(np.packbits(OM.rects_to_bool(pairs, H)), G["tp_single_%d_%s" % (H, r)])
    triples = OT.mask_set_rects(H, r, 2)
    assert len(triples) == 22680
    occluded = np.array([_occluded_count(t, H) for t in triples], np.int32)
    assert np.array_equal(occluded, G["tp_double_sum_%d_%s" % (H, r)])
    probes = OM.rects_to_bool([triples[k] for k in G["tp_probes"]], H)
    assert np.array_equal(np.packbits(probes), G["tp_double_probe_%d_%s" % (H, r)])


def _occluded_count(rects, H):
    m = np.zeros((H, H), bool)
    for r0, r1, c0, c1 in rects:
        m[r0:r1, c0:c1] = True
    return int(m.sum())


def test_fixture_geometry_at_224():
    """The two-patch window at r is the one-patch window at r/2 (mask, stride, window)."""
    want = {0.015: (19, 35, 53), 0.03: (27, 33, 59), 0.06: (38, 32, 69), 0.12: (54, 29, 82)}
    for r, g in want.items():
        assert tuple(G["tp_geom_224_%s" % r]) == g


def test_fixture_covers_both_rounds():
    """At least one stored record takes the second round (round 1 not unanimous), at least one does not."""
    split = [len(np.unique(G["tp_rec_%s_%d_p1" % (r, k)])) > 1 for r in MG.RECORD_RATIOS for k in range(len(MG.SEEDS))]
    assert any(split) and not all(split)
    assert len(G["tp_probes"]) >= 5 and {0, 629, 630, 22679} <= set(G["tp_probes"].tolist())


def _check_record(got, r, k):
    pred, cert, p1, p2 = got
    assert [int(pred), int(cert)] == list(G["tp_rec_%s_%d_pred" % (r, k)])
    assert np.array_equal(np.asarray(p1).astype(np.int64), G["tp_rec_%s_%d_p1" % (r, k)])
    assert np.array_equal(np.packbits(np.asarray(p2).astype(bool)), G["tp_rec_%s_%d_p2" % (r, k)])


@pytest.mark.parametrize("r", MG.RECORD_RATIOS)
def test_oracle_two_patch_records_match_reference(r):
    tiny = _tiny()
    for k, s in enumerate(MG.SEEDS):
        _check_record(OT.robust_predict(tiny, MG.two_patch_image(s), 56, r, certify=True), r, k)


@pytest.mark.parametrize("H", [56, 112, 224])
@pytest.mark.parametrize("r", RATIOS)
def test_product_tables_equal_oracle(H, r):
    for dropout, shape in ((1, (630, 2, 4)), (2, (22680, 3, 4))):
        got = PM.mask_set(H, r, dropout, n_patch=2)
        assert got.shape == shape and got.dtype == np.int16
        assert np.array_equal(got, OT.rects_to_array(OT.mask_set_rects(H, r, dropout)))


@pytest.mark.parametrize("r", [0.03, 0.06, 0.12])
def test_two_patch_window_is_one_patch_pairs_at_half_ratio(r):
    two, one = _mask_window(224, r, 2), _mask_window(224, r / 2, 1)
    assert np.array_equal(two.mask_rects, one.double_mask_rects)
    assert (two.mask_size, two.stride, two.window_size) == (one.mask_size, one.stride, one.window_size)


def test_mask_window_n_patch_3_raises():
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow
    with pytest.raises(NotImplementedError):
        MaskWindow(224, 0.03, 3)
    with pytest.raises(NotImplementedError):
        PM.mask_set(224, 0.03, 1, n_patch=3)


def test_mask_window_prints_two_patch_geometry():
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        mw = MaskWindow(224, 0.12, 2)
    assert buf.getvalue().strip() == "mask size: 54, window size: 82, stride: 29"
    assert mw.n_patch == 2 and mw.mask_rects.shape == (630, 2, 4) and mw.double_mask_rects.shape == (22680, 3, 4)
    assert mw._bool == {}                     # the 1.1 GB bool double_mask_set is built only when read


def test_pc_n_patch_flag_stays_out_of_the_result_path(tmp_path, monkeypatch):
    from dorpatch_b200.main import parser
    from dorpatch_b200.utils import generate_saving_path
    monkeypatch.chdir(tmp_path)
    base = ["--synthetic", "2", "--random_init", "--img_size", "112"]
    default, two = parser.parse_args(base), parser.parse_args(base + ["--pc_n_patch", "2"])
    assert default.pc_n_patch == 1 and two.pc_n_patch == 2
    with pytest.raises(SystemExit), contextlib.redirect_stderr(io.StringIO()):
        parser.parse_args(base + ["--pc_n_patch", "3"])
    with contextlib.redirect_stdout(io.StringIO()):
        assert generate_saving_path(vars(default).copy()) == generate_saving_path(vars(two).copy())


def test_gather_on_pair_tables_is_unchanged():
    """k = 2 tables (the attack's universe, the one-patch window): rectangles in slots 0-1, idx_dual's in slots 2-3."""
    table = PM.universe(112, 2)
    rng = np.random.RandomState(0)
    idx, idx2 = rng.randint(0, len(table), (3, 5)), rng.randint(0, len(table), (3, 5))
    want = np.zeros((3, 5, 4, 4), np.int16)
    want[..., 0:2, :] = table[idx]
    assert PM.gather(table, idx).tobytes() == want.tobytes()
    want[..., 2:4, :] = table[idx2]
    assert PM.gather(table, idx, idx2).tobytes() == want.tobytes()


def test_gather_on_triple_tables():
    table = PM.mask_set(112, 0.06, 2, n_patch=2)
    idx = np.array([0, 17 * 630 + 5, 22679])
    got = PM.gather(table, idx)
    assert got.shape == (3, 4, 4) and got.dtype == np.int16
    assert np.array_equal(got[:, 0:3], table[idx]) and not got[:, 3].any()
    with pytest.raises(ValueError):
        PM.gather(table, idx, idx)


class _TinyPatchCleanser:
    """PatchCleanser.robust_predict over its own rectangle tables, with the classifier replaced by TinyNet on the CPU
    (occlude the image with each sample's <= 4 rectangles, then argmax) -- its control flow, tables and round-2
    construction are what the test checks against the reference."""

    def __init__(self, mw):
        from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
        from dorpatch_b200.resnetv2 import ResNetV2
        self.calls = []
        self.tiny = _tiny()
        self.pc = PatchCleanser(mw, ResNetV2())
        self.pc._predict = self._predict

    def _predict(self, img, rects):
        self.calls.append(rects.copy())
        keep = torch.from_numpy(PM.to_bool(rects, img.shape[-1]))
        # the reference certifies in batches of 64 (PatchCleanser.py:107-109); every other call is one batch
        bs = 64 if len(rects) == len(self.pc.mask_window.double_mask_rects) else len(rects)
        with torch.no_grad():
            out = [self.tiny(img * keep[i:i + bs] + 0.5 * ~keep[i:i + bs]).argmax(1) for i in range(0, len(rects), bs)]
        return torch.cat(out).numpy().astype(np.int32)


@pytest.mark.parametrize("r", MG.RECORD_RATIOS)
def test_robust_predict_two_patch_matches_reference(r):
    for k, s in enumerate(MG.SEEDS):
        t = _TinyPatchCleanser(_mask_window(56, r, 2))
        rec = t.pc.robust_predict(MG.two_patch_image(s), True)
        _check_record((rec.prediction, rec.certification, rec.preds_1, rec.preds_2), r, k)
        assert rec.preds_1.shape == (630,) and rec.preds_2.shape == (22680,)
        n1 = t.calls[0]
        assert n1.shape == (630, 4, 4) and not n1[:, 2:].any()
        for c in t.calls[1:-1]:               # round 2: every pair j plus the disagreeing pair in slots 2-3
            assert c.shape == (630, 4, 4) and np.array_equal(c[:, 0:2], n1[:, 0:2])
            assert (c[:, 2:4] == c[0, 2:4]).all() and any(np.array_equal(c[0, 2:4], n1[j, 0:2]) for j in range(630))
        assert t.calls[-1].shape == (22680, 4, 4)


def test_robust_predict_one_patch_issues_the_same_calls():
    """n_patch 1: round 1 over the 36 singles, one 36-sample call per disagreeing single with it in slot 2, then the
    630-pair certificate -- the tables and batch sizes the one-patch evaluation has always used."""
    img = MG.two_patch_image(1158)
    t = _TinyPatchCleanser(_mask_window(56, 0.12, 1))
    rec = t.pc.robust_predict(img, True)
    single = np.zeros((36, 4, 4), np.int16)
    single[:, 0] = OM.rects_to_array(OM.mask_set_rects(56, 0.12, 1))[:, 0]
    assert np.array_equal(t.calls[0], single)
    labels, counts = torch.from_numpy(rec.preds_1).unique(sorted=False, return_counts=True)
    majority = labels[counts.argmax()].item()
    assert len(labels) > 1                    # this image takes the second round
    want = []
    for label in labels.tolist():
        if label != majority:
            for k in np.nonzero(rec.preds_1 == label)[0]:
                w = single.copy()
                w[:, 2] = single[k, 0]
                want.append(w)
    double = np.zeros((630, 4, 4), np.int16)
    double[:, 0:2] = OM.rects_to_array(OM.mask_set_rects(56, 0.12, 2))
    want.append(double)
    assert len(t.calls) == 1 + len(want)
    for got, w in zip(t.calls[1:], want):
        assert got.dtype == np.int16 and np.array_equal(got, w)
