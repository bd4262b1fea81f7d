"""Golden trajectories of the reference's DorPatch.generate at basic_units other than the default 7, produced by running
the UNMODIFIED reference (located by DORPATCH_REFERENCE_ROOT) under the CPU shim of oracle/ref_shim.py, like
make_golden.py; the fixture is committed next to this script, so the tests need no reference checkout.

    DORPATCH_REFERENCE_ROOT=/path/to/DorPatch python tests/golden/make_basic_unit_golden.py

`basic_unit` sets the side of the square cells of the group lasso (reference attack.py:72-74,243-245) and of
patch_selection (:363-382).  Every run is TinyNet (make_golden.py) at 56 px on make_golden's G6 image, 250 iterations
per stage (past the i > 200 coefficient adaptation), dropout 1:
  u1   basic_unit=1:  per-pixel groups; every pixel clipped to exactly 0 is an all-zero group (NaN gradient, sign 0)
  u4   basic_unit=4:  groups that straddle the 7-px density windows
  u14  basic_unit=14: groups larger than a density window

Writes reference_golden_basic_unit.npz (< 1 MB):
  bu_x                      the image
  bu_<run>_{mask,pattern}   final mask (packbits when binary) and pattern
  bu_<run>_log              every printed line except MaskWindow's "mask size" lines
  bu_<run>_rng_np / _rng_t  numpy legacy-RNG state words and the next three torch.rand draws afterwards
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

OUT = "reference_golden_basic_unit.npz"
# y_shift: targeted at (clean label + y_shift) % 1000.  Every run is targeted: an untargeted reference run that stays
# untargeted through stage 0 stops at its end on set_target(preds_adv), called without its label (attack.py:359).
RUNS = {
    "u1": dict(basic_unit=1, patch_budget=0.12, y_shift=5, max_iterations=250, sampling_size=8, dropout=1),
    "u4": dict(basic_unit=4, patch_budget=0.10, y_shift=3, max_iterations=250, sampling_size=8, dropout=1),
    "u14": dict(basic_unit=14, patch_budget=0.12, y_shift=5, max_iterations=250, sampling_size=8, dropout=1),
}


def _make_golden():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def image():
    """make_golden's G6 image [1,3,56,56]."""
    return torch.rand(1, 3, 56, 56, generator=torch.Generator().manual_seed(5))


def run_kwargs(name, tiny, x):
    kw = dict(RUNS[name])
    shift = kw.pop("y_shift")
    if shift is not None:
        with torch.no_grad():
            kw["y"] = (tiny(x).argmax(-1) + shift) % 1000
    kw["targeted"] = shift is not None
    return kw


def main():
    torch.set_num_threads(8)
    MG = _make_golden()
    tiny = MG.TinyNet().eval()
    x = image()
    out = {"bu_x": x.numpy()}
    with ref_shim.reference_modules() as ref:
        for name in RUNS:
            mo, po, log, rn, rt = MG.run_generate(ref, tiny, x, n_classes=1000, **run_kwargs(name, tiny, x))
            out["bu_%s_mask" % name] = np.packbits(mo.astype(bool)) if set(np.unique(mo)) <= {0.0, 1.0} else mo
            out["bu_%s_pattern" % name] = po
            out["bu_%s_log" % name] = np.array(log)
            out["bu_%s_rng_np" % name] = rn
            out["bu_%s_rng_t" % name] = rt
            print(name, "log lines", len(log), "mask mean", mo.mean())
    path = os.path.join(HERE, OUT)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))
    assert os.path.getsize(path) < 1 << 20


def load():
    with np.load(os.path.join(HERE, OUT), allow_pickle=False) as f:
        return {k: f[k] for k in f.files}


if __name__ == "__main__":
    main()
