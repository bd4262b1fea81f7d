"""Oracle: the two-patch PatchCleanser window and its defense.

Restates reference defenses/PatchCleanser.py:11-16 and :31-37 with n_patch=2
(MaskWindow: geometry, ``mask_set``, ``double_mask_set``) and :68-112
(robust_predict, robustness_certificate) over those sets.  A mask is a tuple of
axis-aligned rectangles (r0, r1, c0, c1), rows [r0,r1) x cols [c0,c1)
occluded: two for ``mask_set``, three for ``double_mask_set``.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import math

import numpy as np
import torch

from . import masks as omasks
from .attack import occlude

N_PATCH = 2


def window_geometry(img_size, patch_ratio):
    """(mask_size, stride, window_size) -- PatchCleanser.py:11-16 with n_patch=2."""
    return omasks.window_geometry(img_size, patch_ratio, N_PATCH)


def basic_rects(img_size, patch_ratio):
    """The 36 basic rectangles of the two-patch geometry; k=i*6+j starts at row
    stride*i, col stride*j -- PatchCleanser.py:44-59."""
    _, stride, window = window_geometry(img_size, patch_ratio)
    rects = []
    for i in range(omasks.N_AXIS):
        for j in range(omasks.N_AXIS):
            r0, c0 = stride * i, stride * j
            rects.append((r0, min(img_size, r0 + window), c0, min(img_size, c0 + window)))
    return rects


def mask_set_rects(img_size, patch_ratio, dropout):
    """dropout=1 (``mask_set``, PatchCleanser.py:23-29,35): the 630 pairs, in
    the order of masks.double_pairs.  dropout=2 (``double_mask_set``, :36-37):
    (combined_mask[None, :] * basic_mask[:, None]) flattened, i.e. mask
    i*630+j is the triple (pair j's two rectangles, basic rectangle i); i in
    pair j is kept."""
    basic = basic_rects(img_size, patch_ratio)
    pairs = [(basic[a], basic[b]) for a, b in omasks.double_pairs()]
    if dropout == 1:
        return pairs
    if dropout == 2:
        return [pair + (b,) for b in basic for pair in pairs]
    raise ValueError("dropout must be 1 or 2")


def rects_to_array(masks):
    """-> int16 [n, k, 4], k = rectangles per mask."""
    return np.asarray(masks, dtype=np.int16).reshape(len(masks), len(masks[0]), 4)


def robust_predict(model, img, img_size, patch_ratio, certify=True, batch_size=64):
    """img [3,H,W] -> (prediction, certification, preds_1[630], preds_2[22680] or None)."""
    singles = torch.from_numpy(omasks.rects_to_bool(mask_set_rects(img_size, patch_ratio, 1), img_size))
    doubles = torch.from_numpy(omasks.rects_to_bool(mask_set_rects(img_size, patch_ratio, 2), img_size))

    def certificate(label):                                   # PatchCleanser.py:102-112
        preds = []
        for i in range(math.ceil(len(doubles) / batch_size)):
            preds.append(model(occlude(img, doubles[i * batch_size:(i + 1) * batch_size])).argmax(1))
        consistent = torch.cat(preds) == label
        return bool(consistent.all().item()), consistent

    with torch.no_grad():
        masked = occlude(img, singles)                        # :70
        preds_1 = model(masked).argmax(1)                     # :72
        labels, counts = preds_1.unique(sorted=False, return_counts=True)   # :74
        majority = labels[counts.argmax()].item()             # :75
        pred, preds_2 = majority, None
        if len(labels) == 1:                                  # :78-79
            certifiable, preds_2 = certificate(pred)
        else:                                                 # :80-90
            certifiable = False
            for label in labels:
                if label == majority:
                    continue
                for masked_img in masked[preds_1 == label]:
                    p12 = model(occlude(masked_img, singles)).argmax(-1)
                    if (p12 == label).all():
                        pred = label.item()
        if certify and preds_2 is None:                       # :93-94
            preds_2 = certificate(majority)[1]
    return pred, certifiable, preds_1.numpy(), (None if preds_2 is None else preds_2.numpy())
