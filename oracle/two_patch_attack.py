"""Oracle: DorPatch.generate trained against the two-patch PatchCleanser window.

The reference's generate always builds its mask universe with get_mask_set, i.e.
MaskWindow(img_size, dropout_size) with n_patch=1 (reference attack.py:25-31,83-85).
``generate(..., pc_n_patch=2)`` is oracle/attack.py's generate with that universe
drawn from MaskWindow(img_size, dropout_size, 2) instead (oracle/two_patch.py):
dropout=1 its 630 pairs per ratio, dropout=2 its 22 680 three-rectangle masks per
ratio.  Nothing else changes: sampling, scans, bookkeeping and RNG consumption are
oracle/attack.py's.  The reference fixture for it (tests/golden/
make_two_patch_attack_golden.py) makes the same single substitution in the
unmodified reference.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
from . import attack as oattack
from . import masks as omasks
from . import two_patch


def universe_rects(img_size, dropout, sizes=omasks.DROPOUT_SIZES):
    """The two-patch universe as rectangle tuples: concat over the four dropout sizes."""
    return [m for r in sizes for m in two_patch.mask_set_rects(img_size, r, dropout)]


def generate(model, x, patch_budget, n_classes, pc_n_patch=1, **kw):
    """oracle/attack.py generate; pc_n_patch=2 swaps the universe for the two-patch window's."""
    if pc_n_patch == 1:
        return oattack.generate(model, x, patch_budget, n_classes, **kw)
    if pc_n_patch != 2:
        raise NotImplementedError("pc_n_patch=%r" % (pc_n_patch,))
    one_patch = omasks.universe_rects
    omasks.universe_rects = universe_rects          # the one name oracle/attack.py builds its universe from
    try:
        return oattack.generate(model, x, patch_budget, n_classes, **kw)
    finally:
        omasks.universe_rects = one_patch
