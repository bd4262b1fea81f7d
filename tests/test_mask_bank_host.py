"""Host-side checks of the mask-bank occlusion (no GPU needed): packing bool keep-masks into the bank layout and back,
the C entry points' declarations, and the errors raised before any engine is built."""
import os
import re

import numpy as np
import pytest
import torch

from dorpatch_b200 import masks as PM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("dp_expand_bank", "dp_predict_bank", "dp_eot_forward_bank", "dp_debug_stem_bwd_reduce_bank")


def _random_keep(M, H, W, seed):
    rng = np.random.RandomState(seed)
    keep = rng.rand(M, 1, H, W) > 0.3
    keep[0] = True                                              # occludes nothing
    keep[1] = False                                             # occludes everything
    keep[2, 0, :, W - 1] = False                                # the last column only
    return keep


@pytest.mark.parametrize("H,W", [(112, 112), (224, 224), (56, 100), (8, 33), (4, 31)])
def test_pack_unpack_round_trip(H, W):
    keep = _random_keep(5, H, W, H + W)
    bank = PM.pack_bank(keep, device="cpu")
    assert bank.dtype == torch.int32 and bank.shape == (5, H, PM.bank_words(W)) and bank.is_contiguous()
    assert np.array_equal(PM.unpack_bank(bank, W).numpy(), keep)
    assert np.array_equal(PM.unpack_bank(PM.pack_bank(torch.from_numpy(keep[:, 0]), device="cpu"), W).numpy(), keep)
    assert (bank[0] == 0).all()                                 # all kept: no bit set
    occ = ~keep[:, 0]                                           # bit w % 32 of word w / 32 = pixel w occluded
    h, w = 3 % H, W - 1
    word = int(bank[4, h, w // 32]) & 0xffffffff
    assert bool((word >> (w % 32)) & 1) == bool(occ[4, h, w])
    if W % 32:                                                  # padding bits past the last column stay clear
        assert (bank[1, :, -1].numpy().astype(np.int64) & 0xffffffff == (1 << (W % 32)) - 1).all()


def test_pack_bank_matches_rectangles():
    table = PM.universe(112, 2)[:50]
    keep = PM.to_bool(table, 112)
    assert np.array_equal(PM.unpack_bank(PM.pack_bank(keep, device="cpu"), 112).numpy(), keep)


def test_pack_bank_refuses_bad_input():
    with pytest.raises(TypeError):
        PM.pack_bank(np.zeros((2, 1, 8, 8), np.float32), device="cpu")
    with pytest.raises(ValueError):
        PM.pack_bank(np.zeros((2, 3, 8, 8), bool), device="cpu")
    with pytest.raises(ValueError):
        PM.pack_bank(np.zeros((8, 8), bool), device="cpu")


def test_bank_entry_points_declared():
    from dorpatch_b200 import _lib
    header = open(os.path.join(ROOT, "include", "dorpatch.h")).read()
    assert int(re.search(r"#define DP_ABI_VERSION (\d+)", header).group(1)) == 9 == _lib.ABI_VERSION
    for name in NEW_SYMBOLS:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib.SIGNATURES, name
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        for name in NEW_SYMBOLS:
            assert getattr(lib, name).argtypes is not None


def _model():
    from dorpatch_b200.resnetv2 import ResNetV2
    return ResNetV2(num_classes=10, seed=0)


def test_eot_logits_bank_refusals_before_any_engine():
    from dorpatch_b200.ops import eot_logits
    net = _model()
    x = torch.rand(2, 3, 56, 56)
    bank = PM.pack_bank(np.ones((3, 1, 56, 56), bool), device="cpu")
    rects = np.zeros((2, 2, 4, 4), np.int16)
    with pytest.raises(ValueError, match="not both"):
        eot_logits(net, x, rects, S=2, bank=bank, idx=np.zeros((2, 2), np.int64))
    with pytest.raises(ValueError, match="xforms"):
        eot_logits(net, x, S=2, xforms=np.zeros((2, 2, 8), np.float32), bank=bank, idx=np.zeros((2, 2), np.int64))
    with pytest.raises(ValueError, match="outside"):
        eot_logits(net, x, S=2, bank=bank, idx=np.full((2, 2), 3))
    with pytest.raises(ValueError, match="outside"):
        eot_logits(net, x, S=2, bank=bank, idx=np.full((2, 2, 2), -2))
    with pytest.raises(ValueError, match="idx"):
        eot_logits(net, x, S=2, bank=bank, idx=None)
    with pytest.raises(ValueError, match=r"\[B, S\]"):
        eot_logits(net, x, S=2, bank=bank, idx=np.zeros((2, 3), np.int64))
    with pytest.raises(TypeError):
        eot_logits(net, x, S=2, bank=bank, idx=np.zeros((2, 2), np.float32))
    with pytest.raises(TypeError):
        eot_logits(net, x, S=2, bank=bank.float(), idx=np.zeros((2, 2), np.int64))
    with pytest.raises(ValueError, match="without a bank"):
        eot_logits(net, x, S=1, idx=np.zeros((2, 1), np.int64))
    with pytest.raises(RuntimeError, match="CUDA"):                # valid arguments: only then the device check
        eot_logits(net, x, S=2, bank=bank, idx=np.zeros((2, 2), np.int64))
    assert net._engines == {}
