"""Golden trajectories of the reference's DorPatch.generate trained against the two-patch PatchCleanser window, produced
by running the UNMODIFIED reference (located by DORPATCH_REFERENCE_ROOT) under the CPU shim of oracle/ref_shim.py, like
make_golden.py; the fixture is committed next to this script, so the tests need no reference checkout.

    DORPATCH_REFERENCE_ROOT=/path/to/DorPatch python tests/golden/make_two_patch_attack_golden.py

The reference's generate builds its universe with attack.get_mask_set, which always uses the one-patch window
(reference attack.py:25-31,83-85).  The single change made here is to swap get_mask_set for a function returning the
reference's own MaskWindow(img_size, dropout_size, 2).mask_set (dropout 1) / .double_mask_set (dropout 2).

Writes reference_golden_two_patch_attack.npz (< 1 MB), TinyNet (make_golden.py) at 56 px on make_golden's G6 image:
  tpa_x                      the image
  tpa_<run>_{mask,pattern}   final mask (packbits when binary) and pattern
  tpa_<run>_log              every printed line except MaskWindow's "mask size" lines
  tpa_<run>_rng_np / _rng_t  numpy legacy-RNG state words and the next three torch.rand draws afterwards
Runs (RUNS): d1 -- dropout 1, the 2 520 pairs; d2 -- dropout 2, the 90 720 three-rectangle masks, reaching i >= 1000
with a non-empty failed set so that the samples drawn from the failed set come from the two-patch universe.
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

OUT = "reference_golden_two_patch_attack.npz"
# y_shift: targeted at (clean label + y_shift) % 1000, None = untargeted
RUNS = {
    "d1": dict(patch_budget=0.12, y_shift=5, max_iterations=250, sampling_size=8, dropout=1),
    "d2": dict(patch_budget=0.10, y_shift=None, max_iterations=1020, sampling_size=16, dropout=2),
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


def failed_at_1000(log):
    """Failed-set sizes of the scans at i == 1000 (the line printed right before 'iteration: 1000')."""
    return [int(log[k - 1].split()[1]) for k, l in enumerate(log) if l.startswith("iteration: 1000,")]


def main():
    torch.set_num_threads(8)
    MG = _make_golden()
    tiny = MG.TinyNet().eval()
    x = image()
    out = {"tpa_x": x.numpy()}
    with ref_shim.reference_modules() as ref:
        PC = ref.PatchCleanser

        def two_patch_mask_set(img_size, dropout_size, dropout):
            mw = PC.MaskWindow(img_size, dropout_size, 2)
            return mw.mask_set if dropout == 1 else (mw.double_mask_set if dropout == 2 else None)

        ref.attack.get_mask_set = two_patch_mask_set
        for name in RUNS:
            mo, po, log, rn, rt = MG.run_generate(ref, tiny, x, n_classes=1000, **run_kwargs(name, tiny, x))
            out["tpa_%s_mask" % name] = np.packbits(mo.astype(bool)) if set(np.unique(mo)) <= {0.0, 1.0} else mo
            out["tpa_%s_pattern" % name] = po
            out["tpa_%s_log" % name] = np.array(log)
            out["tpa_%s_rng_np" % name] = rn
            out["tpa_%s_rng_t" % name] = rt
            print(name, "log lines", len(log), "mask mean", mo.mean(), "failed at i=1000", failed_at_1000(log))
    assert any(n > 0 for n in failed_at_1000(list(out["tpa_d2_log"]))), "d2 never samples from a non-empty failed set"
    assert not failed_at_1000(list(out["tpa_d1_log"]))
    path = os.path.join(HERE, OUT)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))
    assert os.path.getsize(path) < 1 << 20


def load():
    with np.load(os.path.join(HERE, OUT), allow_pickle=False) as f:
        return {k: f[k] for k in f.files}


if __name__ == "__main__":
    main()
