"""Oracle: PatchCleanser occlusion-mask geometry as rectangles.

Restates reference defenses/PatchCleanser.py:8-59 (MaskWindow) and the
attack's mask universe (reference attack.py:25-31,83-85).
Every mask is "keep everything except <= 2 axis-aligned rectangles" (True=keep).
A rectangle is (r0, r1, c0, c1), rows [r0,r1) x cols [c0,c1) occluded.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import math

import numpy as np

DROPOUT_SIZES = (0.015, 0.03, 0.06, 0.12)   # attack.py:83 / main.py:61
N_AXIS = 6                                   # PatchCleanser.py:13
EMPTY = (0, 0, 0, 0)


def window_geometry(img_size, patch_ratio, n_patch=1):
    """(mask_size, stride, window_size) -- PatchCleanser.py:11-16."""
    mask_size = math.floor(math.sqrt(img_size ** 2 * patch_ratio / n_patch))
    stride = int(np.ceil((img_size - mask_size + 1) / N_AXIS))
    window = mask_size + stride - 1
    return mask_size, stride, window


def single_rects(img_size, patch_ratio):
    """36 rectangles; mask k=i*6+j occludes rows from stride*i, cols from
    stride*j -- PatchCleanser.py:44-59 (dim 2 = rows is indexed by i)."""
    _, stride, window = window_geometry(img_size, patch_ratio)
    rects = []
    for i in range(N_AXIS):
        for j in range(N_AXIS):
            r0, c0 = stride * i, stride * j
            rects.append((r0, min(img_size, r0 + window), c0, min(img_size, c0 + window)))
    return rects


def double_pairs(n=N_AXIS * N_AXIS):
    """Upper-triangular (a<b) pairs in row-major order -- PatchCleanser.py:21-29."""
    return [(a, b) for a in range(n) for b in range(a + 1, n)]


def mask_set_rects(img_size, patch_ratio, dropout):
    """Rect pairs [(rectA, rectB)] for ``mask_set`` (dropout=1, rectB empty) or
    ``double_mask_set`` (dropout=2) -- attack.py:25-31."""
    singles = single_rects(img_size, patch_ratio)
    if dropout == 1:
        return [(r, EMPTY) for r in singles]
    if dropout == 2:
        return [(singles[a], singles[b]) for a, b in double_pairs()]
    raise ValueError("dropout must be 1 or 2")


def universe_rects(img_size, dropout, sizes=DROPOUT_SIZES):
    """attack.py:83-85: concat over the four dropout sizes."""
    out = []
    for r in sizes:
        out.extend(mask_set_rects(img_size, r, dropout))
    return out


def rects_to_array(rect_pairs):
    """-> int16 [n, 2, 4] (r0, r1, c0, c1)."""
    return np.asarray(rect_pairs, dtype=np.int16).reshape(len(rect_pairs), 2, 4)


def rects_to_bool(rect_pairs, img_size):
    """Materialise bool masks [n,1,H,W], True = keep."""
    m = np.ones((len(rect_pairs), 1, img_size, img_size), dtype=bool)
    for k, pair in enumerate(rect_pairs):
        for (r0, r1, c0, c1) in pair:
            m[k, 0, r0:r1, c0:c1] = False
    return m
