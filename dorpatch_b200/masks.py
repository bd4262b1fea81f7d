"""Occlusion-mask geometry of the PatchCleanser mask window, as rectangle tables.

Every mask the reference materialises as a [1,H,W] bool tensor
(reference defenses/PatchCleanser.py:8-59, reference attack.py:25-31,83-85) is
"keep everything except <= 3 axis-aligned rectangles" (<= 2 for the one-patch window and the
attack's universe, 3 for the two-patch window's double masks); the native K1 kernel synthesises
the occlusion from up to 4 rectangles per sample (int16 r0,r1,c0,c1 -- rows [r0,r1) x cols
[c0,c1) become 0.5), so the 126 MB bool universe (1.1 GB for the two-patch double masks at
224 px) is never built.
"""
import math

import numpy as np

DROPOUT_SIZES = (0.015, 0.03, 0.06, 0.12)
MASKS_PER_AXIS = 6


class WindowGeometry:
    """mask_size / stride / window_size of one patch ratio (PatchCleanser.py:11-16)."""

    def __init__(self, img_size, patch_ratio, n_patch=1):
        self.img_size = int(img_size)
        self.mask_size = math.floor(math.sqrt(img_size ** 2 * patch_ratio / n_patch))
        self.stride = int(np.ceil((img_size - self.mask_size + 1) / MASKS_PER_AXIS))
        self.window_size = self.mask_size + self.stride - 1

    def single_rects(self):
        """int16 [36,4]: mask k = i*6+j starts at row stride*i, col stride*j."""
        k = np.arange(MASKS_PER_AXIS)
        lo = self.stride * k
        hi = np.minimum(self.img_size, lo + self.window_size)
        r = np.zeros((MASKS_PER_AXIS, MASKS_PER_AXIS, 4), np.int16)
        r[:, :, 0], r[:, :, 1] = lo[:, None], hi[:, None]
        r[:, :, 2], r[:, :, 3] = lo[None, :], hi[None, :]
        return r.reshape(-1, 4)


def pair_index():
    """(a,b), a<b, row-major over the 36x36 upper triangle (PatchCleanser.py:21-29)."""
    a, b = np.triu_indices(MASKS_PER_AXIS ** 2, k=1)
    return a, b


def mask_set(img_size, patch_ratio, dropout, n_patch=1):
    """Rectangle table of `mask_set` (dropout 1) / `double_mask_set` (dropout 2) of the window for n_patch patches
    (PatchCleanser.py:19-39).  n_patch 1: int16 [36,2,4] single rectangles (slot 1 empty) / [630,2,4] pairs.
    n_patch 2 (36 basic rectangles of the two-patch geometry): [630,2,4] pairs / [22680,3,4], mask i*630+j = pair j
    plus basic rectangle i (PatchCleanser.py:36-37; entries with i in pair j are kept, as there)."""
    if n_patch == 2:
        return _two_patch_set(img_size, patch_ratio, dropout)
    if n_patch != 1:
        raise NotImplementedError("n_patch=%r: PatchCleanser masks exist for 1 or 2 patches" % (n_patch,))
    s = WindowGeometry(img_size, patch_ratio).single_rects()
    if dropout == 1:
        out = np.zeros((len(s), 2, 4), np.int16)
        out[:, 0] = s
        return out
    if dropout == 2:
        a, b = pair_index()
        return np.stack([s[a], s[b]], axis=1)
    raise ValueError("dropout must be 1 or 2, got %r" % (dropout,))


def _two_patch_set(img_size, patch_ratio, dropout):
    s = WindowGeometry(img_size, patch_ratio, 2).single_rects()
    a, b = pair_index()
    pairs = np.stack([s[a], s[b]], axis=1)                     # [630,2,4]
    if dropout == 1:
        return pairs
    if dropout == 2:
        out = np.empty((len(s), len(pairs), 3, 4), np.int16)   # [basic i, pair j]
        out[:, :, 0:2] = pairs[None]
        out[:, :, 2] = s[:, None]
        return out.reshape(-1, 3, 4)
    raise ValueError("dropout must be 1 or 2, got %r" % (dropout,))


def universe(img_size, dropout, n_patch=1, sizes=DROPOUT_SIZES):
    """The attack's mask universe (attack.py:83-85) drawn from the window for n_patch patches: the concatenation over
    the four ratios of mask_set(img_size, r, dropout, n_patch).  n_patch 1: [144,2,4] / [2520,2,4]; n_patch 2:
    [2520,2,4] / [90720,3,4], mask r*22680 + i*630 + j as in the reference's double_mask_set."""
    return np.concatenate([mask_set(img_size, r, dropout, n_patch) for r in sizes], axis=0)


def distinct_occlusions(table, n_sets=1):
    """The distinct occlusions of a rectangle table [n,k,4] and the map back: (distinct [m,k,4], inv [n]) with
    table[k] and distinct[inv[k]] occluding the same pixels.  The table is the concatenation of n_sets equally long
    mask sets (the universe: one per ratio); two masks are the same occlusion when they lie in the same set and list
    the same basic rectangles (order and repeats ignored).  distinct[j] is the first such mask of the table, and
    distinct keeps the table's order, so a table without repeats maps to itself (inv = arange(n)).  The two-patch
    dropout-2 universe holds each triple {i,a,b} of basic rectangles 3 times and each pair 2 times (mask
    i*630 + pair(a,b) with i in {a,b}): 7 770 distinct occlusions per ratio out of 22 680."""
    t = np.asarray(table).astype(np.int64)
    n = t.shape[0]
    if n % n_sets:
        raise ValueError("a table of %d masks is not %d equally long sets" % (n, n_sets))
    key = (t[..., 0] << 48) | (t[..., 1] << 32) | (t[..., 2] << 16) | t[..., 3]   # one int64 per rectangle; empty = 0
    key = np.sort(key, axis=1)
    key[:, 1:][key[:, 1:] == key[:, :-1]] = 0                                       # a repeated rectangle adds nothing
    key = np.sort(key, axis=1)
    key = np.concatenate([(np.arange(n) // (n // n_sets))[:, None], key], axis=1)  # never merge across sets
    _, first, inv = np.unique(key, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first)
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return np.ascontiguousarray(table[first[order]]), rank[inv.reshape(-1)]


def gather(table, idx, idx_dual=None):
    """Rectangles of the sampled masks: table [n,k,4] (k <= 4), idx [...] -> [...,4,4] int16 with the table's k
    rectangles in slots 0..k-1; slots 2-3 come from idx_dual (k = 2 tables only), else the rest is empty."""
    idx = np.asarray(idx)
    k = table.shape[1]
    if k > 4 or (idx_dual is not None and k > 2):
        raise ValueError("gather: %d-rectangle table%s exceeds the 4 rectangle slots of a sample"
                         % (k, " with idx_dual" if idx_dual is not None else ""))
    out = np.zeros(idx.shape + (4, 4), np.int16)
    out[..., 0:k, :] = table[idx]
    if idx_dual is not None:
        out[..., 2:4, :] = table[np.asarray(idx_dual)]
    return out


def to_bool(table, img_size):
    """Materialise [n,1,H,W] bool masks (True = keep) -- only for API compatibility
    (MaskWindow.mask_set) and tests; the engine never uses it."""
    n = table.shape[0]
    m = np.ones((n, 1, img_size, img_size), dtype=bool)
    for k in range(n):
        for r0, r1, c0, c1 in table[k].reshape(-1, 4):
            m[k, 0, r0:r1, c0:c1] = False
    return m


def from_bool(masks):
    """Inverse of to_bool for API compatibility: bool keep-masks [n,1,H,W] (torch or numpy) -> rectangle table
    [n,2,4] int16.  Each mask's occluded set must be a union of <= 2 axis-aligned rectangles, as the reference
    builds them (PatchCleanser.py:51-58: one rectangle per single mask, the union of two per double mask); anything
    else raises -- the engine has no dense-mask path."""
    m = masks.detach().cpu().numpy() if hasattr(masks, "detach") else np.asarray(masks)
    m = m.reshape(m.shape[0], m.shape[-2], m.shape[-1]).astype(bool)
    out = np.zeros((m.shape[0], 2, 4), np.int16)
    for k in range(m.shape[0]):
        out[k] = _decompose(~m[k], k)
    return out


def _decompose(occ, k=0):
    """occ (bool [H,W]) as a union of <= 2 rectangles.  Work on the coarse grid of rows / columns where the pattern
    changes (<= 5 x 5 cells): the first rectangle starts at the first occluded cell; try each of its extents, the
    second rectangle is then the bounding box of what is left, valid if it lies inside the occluded set."""
    H, W = occ.shape
    out = np.zeros((2, 4), np.int16)
    if not occ.any():
        return out
    rb = [0] + [i for i in range(1, H) if not np.array_equal(occ[i], occ[i - 1])] + [H]
    cb = [0] + [j for j in range(1, W) if not np.array_equal(occ[:, j], occ[:, j - 1])] + [W]
    g = occ[np.ix_(rb[:-1], cb[:-1])]
    a0 = int(np.argmax(g.any(1)))
    b0 = int(np.argmax(g[a0]))
    for a1 in range(a0 + 1, g.shape[0] + 1):
        for b1 in range(b0 + 1, g.shape[1] + 1):
            if not g[a0:a1, b0:b1].all():
                continue
            rest = g.copy()
            rest[a0:a1, b0:b1] = False
            if not rest.any():
                out[0] = (rb[a0], rb[a1], cb[b0], cb[b1])
                return out
            rr, cc = np.nonzero(rest)
            # the second rectangle may overlap the first: grow the remainder's bounding box over occluded cells
            for c0 in range(int(rr.min()), -1, -1):
                for d0 in range(int(cc.min()), -1, -1):
                    c1, d1 = int(rr.max()) + 1, int(cc.max()) + 1
                    if not g[c0:c1, d0:d1].all():
                        continue
                    u = np.zeros_like(g)
                    u[a0:a1, b0:b1] = True
                    u[c0:c1, d0:d1] = True
                    if np.array_equal(u, g):
                        out[0] = (rb[a0], rb[a1], cb[b0], cb[b1])
                        out[1] = (rb[c0], rb[c1], cb[d0], cb[d1])
                        return out
    raise NotImplementedError("mask %d is not a union of <= 2 axis-aligned rectangles" % k)


# ---- mask banks: arbitrary occlusions -------------------------------------------------------------------------------
def bank_words(W):
    """uint32 words per row of a mask bank of width W."""
    return (int(W) + 31) // 32


def pack_bank(keep, device=None):
    """Bool keep-masks [M,1,H,W] or [M,H,W] (torch or numpy; True = keep, as the reference's mask sets) -> the mask
    bank the engine reads: a contiguous int32 CUDA tensor [M, H, ceil(W/32)] holding uint32 words, bit w % 32 of word
    w / 32 of row h set = pixel (h, w) occluded.  Any shape of occluder works (``Engine.predict(bank=...)``,
    ``eot_logits(bank=...)``).  device: the CUDA device (default: the masks' own if they are on one, else the current)."""
    import torch
    m = keep if isinstance(keep, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(keep))
    if m.dim() == 4:
        if m.shape[1] != 1:
            raise ValueError("pack_bank: masks must be [M,1,H,W] or [M,H,W], got %s" % (tuple(m.shape),))
        m = m[:, 0]
    if m.dim() != 3 or m.shape[0] < 1:
        raise ValueError("pack_bank: masks must be [M,1,H,W] or [M,H,W] with M >= 1, got %s" % (tuple(keep.shape),))
    if m.dtype != torch.bool:
        raise TypeError("pack_bank: masks must be bool (True = keep), got %s" % (m.dtype,))
    if device is None:
        device = m.device if m.is_cuda else torch.device("cuda", torch.cuda.current_device())
    M, H, W = m.shape
    nw = bank_words(W)
    out = torch.empty((M, H, nw), dtype=torch.int32, device=device)
    shift = torch.arange(32, device=device, dtype=torch.int64)
    for m0 in range(0, M, 512):                                  # bounded scratch for large universes
        part = m[m0:m0 + 512]
        occ = torch.zeros((part.shape[0], H, nw * 32), dtype=torch.int64, device=device)
        occ[:, :, :W] = (~part).to(device=device, dtype=torch.int64)
        w = (occ.view(-1, H, nw, 32) << shift).sum(-1)
        out[m0:m0 + 512] = torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)
    return out


def unpack_bank(bank, W):
    """Inverse of pack_bank: bank [M,H,ceil(W/32)] (torch int32) -> bool keep-masks [M,1,H,W] on the bank's device."""
    import torch
    M, H, nw = bank.shape
    if nw != bank_words(W):
        raise ValueError("unpack_bank: %d words per row do not hold W=%d" % (nw, W))
    bits = (bank.to(torch.int64)[..., None] >> torch.arange(32, device=bank.device, dtype=torch.int64)) & 1
    return (bits.reshape(M, H, nw * 32)[:, :, :W] == 0)[:, None]
