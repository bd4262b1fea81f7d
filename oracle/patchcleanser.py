"""Oracle restatement of the PatchCleanser defense used to score the attack.

Follows reference defenses/PatchCleanser.py:62-112 (robust_predict,
robustness_certificate).  ``model`` maps [N,3,H,W] in [0,1] -> logits on CPU.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import math

import numpy as np
import torch

from . import masks as omasks
from .attack import occlude


def robust_predict(model, img, img_size, patch_ratio, certify=True, batch_size=64):
    """img [3,H,W] -> (prediction, certification, preds_1[36], preds_2[630] or None)."""
    singles = torch.from_numpy(omasks.rects_to_bool(omasks.mask_set_rects(img_size, patch_ratio, 1), img_size))
    doubles = torch.from_numpy(omasks.rects_to_bool(omasks.mask_set_rects(img_size, patch_ratio, 2), img_size))

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
