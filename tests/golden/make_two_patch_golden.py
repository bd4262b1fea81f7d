"""Golden vectors of the reference's two-patch PatchCleanser window (MaskWindow(img, r, n_patch=2)), produced by
running the UNMODIFIED reference (located by DORPATCH_REFERENCE_ROOT) under the CPU shim of oracle/ref_shim.py, like
make_golden.py; the fixture is committed next to this script, so the tests need no reference checkout.

    DORPATCH_REFERENCE_ROOT=/path/to/DorPatch python tests/golden/make_two_patch_golden.py

Writes reference_golden_two_patch.npz (< 1 MB):
  tp_geom_<H>_<r>          (mask_size, stride, window_size) at 56 and 224 px, the four ratios
  tp_single_56_<r>         packbits of all 630 ``mask_set`` masks (pairs) at 56 px
  tp_double_sum_<H>_<r>    occluded-pixel count of each of the 22 680 ``double_mask_set`` masks
  tp_double_probe_<H>_<r>  packbits of ``double_mask_set[PROBES]``
  tp_rec_<r>_<k>_{pred,p1,p2}  TinyNet robust_predict(img, True) records at 56 px: [prediction, certification],
                           preds_1 (630,) int64, packbits of preds_2 (22 680,) bool; images from two_patch_image(SEEDS[k])
"""
import contextlib
import importlib.util
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

OUT = "reference_golden_two_patch.npz"
RATIOS = (0.015, 0.03, 0.06, 0.12)
RECORD_RATIOS = (0.03, 0.12)
# image seeds: 858 has a wide top-2 margin (round 1 unanimous), 1158 and 563 sit near a TinyNet decision boundary so
# the two-patch masks split round 1 and robust_predict takes the second round
SEEDS = (858, 1158, 563)


def _pair_index(a, b, n=36):
    """Position of pair (a, b), a < b, in the row-major upper-triangle order of ``mask_set``."""
    return a * n - a * (a + 1) // 2 + (b - a - 1)


# double_mask_set index i*630 + j: the first and last masks of the first two basic rows, the last mask, and basic 17
# added to pair (3, 17) (i in pair j: the union is the pair itself; index 0 = basic 0 with pair (0, 1) is one too)
PROBES = (0, 1, 629, 630, 631, 17 * 630 + _pair_index(3, 17), 22679)


def _make_golden():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def two_patch_image(seed, size=56):
    """A flat random colour with 30 % texture: TinyNet's label depends on the colour, so grey occlusions near a
    decision boundary flip it."""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(3, 1, 1, generator=g)
    return (0.7 * c + 0.3 * torch.rand(3, size, size, generator=g)).clamp(0, 1)


def main():
    torch.set_num_threads(8)
    out = {"tp_probes": np.array(PROBES, np.int64), "tp_rec_seeds": np.array(SEEDS, np.int64)}
    tiny = _make_golden().TinyNet().eval()
    with ref_shim.reference_modules() as ref:
        PC = ref.PatchCleanser
        with contextlib.redirect_stdout(io.StringIO()):
            for H in (56, 224):
                for r in RATIOS:
                    mw = PC.MaskWindow(H, r, 2)
                    out["tp_geom_%d_%s" % (H, r)] = np.array([mw.mask_size, mw.stride, mw.window_size])
                    assert tuple(mw.mask_set.shape) == (630, 1, H, H)
                    if H == 56:
                        out["tp_single_%d_%s" % (H, r)] = np.packbits(mw.mask_set.numpy())
                    dm = mw.double_mask_set.numpy()
                    assert dm.shape == (22680, 1, H, H)
                    out["tp_double_sum_%d_%s" % (H, r)] = (~dm).reshape(dm.shape[0], -1).sum(1).astype(np.int32)
                    out["tp_double_probe_%d_%s" % (H, r)] = np.packbits(dm[list(PROBES)])
                    del mw, dm
            round2 = unanimous = 0
            for r in RECORD_RATIOS:
                d = PC.PatchCleanser(PC.MaskWindow(56, r, 2), tiny)
                for k, s in enumerate(SEEDS):
                    with torch.no_grad():
                        rec = d.robust_predict(two_patch_image(s), True)
                    assert rec.preds_1.shape == (630,) and rec.preds_2.shape == (22680,)
                    if len(np.unique(rec.preds_1)) > 1:
                        round2 += 1
                    else:
                        unanimous += 1
                    out["tp_rec_%s_%d_pred" % (r, k)] = np.array([rec.prediction, int(rec.certification)])
                    out["tp_rec_%s_%d_p1" % (r, k)] = rec.preds_1.astype(np.int64)
                    out["tp_rec_%s_%d_p2" % (r, k)] = np.packbits(rec.preds_2.astype(bool))
    assert round2 >= 1 and unanimous >= 1, (round2, unanimous)
    print("records: %d take the second round, %d are unanimous in round 1" % (round2, unanimous))
    path = os.path.join(HERE, OUT)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


def load():
    with np.load(os.path.join(HERE, OUT), allow_pickle=False) as f:
        return {k: f[k] for k in f.files}


if __name__ == "__main__":
    main()
