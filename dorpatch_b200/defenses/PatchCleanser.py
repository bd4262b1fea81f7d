"""PatchCleanser defense (evaluation of the generated patch) on the native forward engine.

Mirrors reference defenses/PatchCleanser.py: MaskWindow :6-59, PatchCleanser :62-118
(robust_predict :68-97, mask :99-100, robustness_certificate :102-112), PatchCleanserRecord
:121-126, PatchCleanserResult :129-134.  Masks are rectangle tables (dorpatch_b200.masks);
the bool mask tensors of the reference are materialised lazily, only if someone reads
``mask_set`` / ``double_mask_set``.

``MaskWindow(img, r, n_patch=2)`` is the two-patch window (reference :31-37): 630 first-round pairs and
22 680 certificate masks of 3 rectangles each.  Its second round puts 4 rectangles on a sample, which is
K1's per-sample limit, so the same code and kernels serve both windows.

A window without rectangle tables (any object with bool ``mask_set`` / ``double_mask_set``, as the reference accepts)
is packed into mask banks (``masks.pack_bank``) and runs the same rounds through ``dp_predict_bank``.

``PatchCleanser(..., shard=True)`` under torch.distributed (world > 1, ``DORPATCH_SHARD`` not ``none``) splits the masked
forwards of ``robust_predict`` over the ranks: round 1 and the certificate in whole chunks of the single-process call
(``attack.sharded_predict``), the second-round checks whole and round-robin (``attack.sharded_checks``).  Every rank
returns the single-process record.  The call is then a collective: every rank must make it, with the same image and
arguments, in the same order.  Without ``shard=True`` (the default) every call is local to its process, whichever ranks
make it.
"""
import math

import numpy as np
import torch

from .. import masks as _masks
from ..attack import _dist, sharded_checks, sharded_predict
from ..utils import unwrap_native


class MaskWindow(object):
    def __init__(self, img_size, patch_ratio=0.03, n_patch=1):
        if n_patch not in (1, 2):
            raise NotImplementedError("n_patch=%r: PatchCleanser masks exist for 1 or 2 patches" % (n_patch,))
        g = _masks.WindowGeometry(img_size, patch_ratio, n_patch)
        self.img_size, self.n_patch = img_size, n_patch
        self.mask_size, self.stride, self.window_size = g.mask_size, g.stride, g.window_size
        self.num_mask_per_axis = _masks.MASKS_PER_AXIS
        # n_patch 1: [36,2,4] / [630,2,4];  n_patch 2: [630,2,4] / [22680,3,4]
        self.mask_rects = _masks.mask_set(img_size, patch_ratio, 1, n_patch)
        self.double_mask_rects = _masks.mask_set(img_size, patch_ratio, 2, n_patch)
        self._bool = {}
        print("mask size: %d, window size: %d, stride: %d" % (self.mask_size, self.window_size, self.stride))

    def _materialise(self, name, table):
        if name not in self._bool:
            t = torch.from_numpy(_masks.to_bool(table, self.img_size))
            self._bool[name] = t.cuda() if torch.cuda.is_available() else t
        return self._bool[name]

    @property
    def mask_set(self):
        return self._materialise("single", self.mask_rects)

    @property
    def double_mask_set(self):
        return self._materialise("double", self.double_mask_rects)

    @property
    def reverse_mask_set(self):
        return ~self.mask_set


class PatchCleanser(object):
    def __init__(self, mask_window, model, result=None, shard=False):
        """shard=True: under a torch.distributed group, robust_predict shares its forwards with the other ranks and is a
        collective (see the module docstring); False keeps every call on this process alone."""
        self.mask_window = mask_window
        self.model = model
        self.result = result
        self.shard = bool(shard)
        self._net = unwrap_native(model)
        self.forwards = 0                        # masked forwards this process ran for this defense

    def _engine(self, img):
        return self._net.engine(img.shape[-1], max_images=1)

    def _predict(self, img, rects):
        """argmax predictions of the classifier on occlude(img, rects[k]); rects [n,4,4]."""
        eng = self._engine(img)
        x = img.reshape(1, 3, img.shape[-2], img.shape[-1]).contiguous().float()
        self.forwards += rects.shape[0]
        return eng.predict(x, rects.shape[0], rects)

    def _predict_bank(self, img, bank, idx):
        """The same on a mask bank: sample k occluded by mask idx[k] (or the pair idx[k, 0], idx[k, 1])."""
        eng = self._engine(img)
        x = img.reshape(1, 3, img.shape[-2], img.shape[-1]).contiguous().float()
        self.forwards += len(idx)
        return eng.predict(x, len(idx), bank=bank, idx=idx)

    def _bank(self, name, img):
        """A window without rectangle tables (any object with bool mask_set / double_mask_set, as the reference
        accepts): its set `name` packed into a mask bank on img's device, when first needed (the doubles only when a
        certificate is asked for, as the reference reads them only then), and kept while the window, the set object
        and the device stay the same."""
        mw = self.mask_window
        masks = getattr(mw, name)
        cache = self.__dict__.setdefault("_bank_cache", {})
        key = (name, str(img.device))
        hit = cache.get(key)
        if hit is None or hit[0] is not mw or hit[1] is not masks:
            hit = (mw, masks, _masks.pack_bank(masks, device=img.device))
            cache[key] = hit
        return hit[2]

    def _group(self):
        """The process group the masked forwards are sharded over (shard=True and attack._dist: world > 1 and
        DORPATCH_SHARD not switched off), or None: this process forwards everything."""
        return _dist() if self.shard else None

    def _chunk(self, img):
        return self._engine(img).chunk

    def robust_predict(self, img, certify=False):
        mw = self.mask_window
        if getattr(mw, "mask_rects", None) is None:
            return self._robust_predict_bank(img, certify)
        single = _masks.gather(mw.mask_rects, np.arange(len(mw.mask_rects)))          # [36 or 630,4,4]

        def check(k):
            # second-round masking of the already-masked image: mask j plus mask k's rectangles
            # (one for n_patch 1, a pair for n_patch 2) in slots 2-3
            second = single.copy()
            second[:, 2:4, :] = single[k, 0:2, :]
            return lambda lo, hi: self._predict(img, second[lo:hi])

        return self._rounds(img, certify, len(single), lambda lo, hi: self._predict(img, single[lo:hi]), check)

    def _robust_predict_bank(self, img, certify):
        """robust_predict for a window given as bool mask sets: the same rounds, tie rules and records, each
        occlusion read from a mask bank; the second round occludes with the pair (mask j, mask k)."""
        singles = self._bank("mask_set", img)
        n = singles.shape[0]

        def check(k):
            pairs = np.stack([np.arange(n), np.full(n, k)], axis=1)
            return lambda lo, hi: self._predict_bank(img, singles, pairs[lo:hi])

        return self._rounds(img, certify, n, lambda lo, hi: self._predict_bank(img, singles, np.arange(lo, hi)), check)

    def _rounds(self, img, certify, n, first, check):
        """The rounds of :68-97 over n first-round samples.  first(lo, hi) forwards first-round samples [lo, hi) as one
        call; check(k)(lo, hi) does the same for the second-round check of first-round sample k.  Under a process group
        (_group) every rank forwards a share, split only at chunk boundaries of the call one process would make (round 1,
        certificate) or as whole checks (round 2), and the labels are gathered, so every rank returns the record one
        process returns; every rank must then call robust_predict with the same arguments.  Without a group, every call
        is the single-process call."""
        dist = self._group()
        chunk = self._chunk(img) if dist else None
        preds_1 = sharded_predict(first, n, chunk, dist)                              # :70-72
        labels, counts = torch.from_numpy(preds_1.astype(np.int64)).unique(sorted=False, return_counts=True)
        label_majority = labels[counts.argmax()].item()                               # :74-75
        pred, preds_2 = label_majority, None
        if len(labels) == 1:                                                          # :78-79
            certifiable, preds_2 = self.robustness_certificate(img, pred)
        else:                                                                         # :80-90
            certifiable = False
            # every minority sample k in the reference's order; no early exit, so the forwards are the reference's
            checks = [(label, k) for label in labels.tolist() if label != label_majority
                      for k in np.nonzero(preds_1 == label)[0]]
            passed = sharded_checks(lambda i: (sharded_predict(check(checks[i][1]), n, chunk) == checks[i][0]).all(),
                                    len(checks), dist)
            for (label, _), ok in zip(checks, passed):                                # the last confirmed label wins
                if ok:
                    pred = label
        if certify and preds_2 is None:                                               # :93-94
            preds_2 = self.robustness_certificate(img, label_majority)[1]
        return PatchCleanserRecord(pred, certifiable, preds_1.astype(np.int64),
                                   None if preds_2 is None else np.asarray(preds_2))

    def mask(self, img, msk):
        return img * msk + 0.5 * ~msk

    def robustness_certificate(self, img, label, batch_size=64):
        """All double-mask predictions (630, or 22 680 for n_patch 2) must equal `label` (:102-112).  `batch_size` is kept
        for signature compatibility; batching is the engine's `chunk`."""
        mw = self.mask_window
        dist = self._group()
        chunk = self._chunk(img) if dist else None
        if getattr(mw, "double_mask_rects", None) is None:
            doubles = self._bank("double_mask_set", img)
            preds = sharded_predict(lambda lo, hi: self._predict_bank(img, doubles, np.arange(lo, hi)),
                                    doubles.shape[0], chunk, dist)
        else:
            rects = _masks.gather(mw.double_mask_rects, np.arange(len(mw.double_mask_rects)))
            preds = sharded_predict(lambda lo, hi: self._predict(img, rects[lo:hi]), len(rects), chunk, dist)
        consistent = preds == label
        return bool(consistent.all()), consistent

    def reset(self):
        self.result = None

    def collect(self, records):
        self.result = PatchCleanserResult(records)


class PatchCleanserRecord(object):
    def __init__(self, pred, certifiable, preds_1, preds_2):
        self.prediction = pred
        self.certification = certifiable
        self.preds_1 = preds_1
        self.preds_2 = preds_2


class PatchCleanserResult(object):
    def __init__(self, records):
        self.predictions = np.stack([r.prediction for r in records])
        self.certifications = np.stack([r.certification for r in records])
        self.predictions_1 = np.stack([r.preds_1 for r in records])
        self.predictions_2 = [r.preds_2 for r in records]
