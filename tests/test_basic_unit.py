"""DorPatch.generate(basic_unit=u) for units other than the default 7, on the CPU: the oracle against the reference's
trajectories at u = 1, 4 and 14, the argument check and the result path."""
import importlib.util
import os
import random

import numpy as np
import pytest
import torch

from oracle import attack as OA

HERE = os.path.dirname(os.path.abspath(__file__))


def _module(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, "golden", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MG = _module("make_golden")
MBU = _module("make_basic_unit_golden")
GB = MBU.load()


def _seed(s=1234):
    random.seed(s)
    torch.manual_seed(s)
    np.random.seed(s)


@pytest.mark.parametrize("name", list(MBU.RUNS))
def test_oracle_reproduces_reference_basic_unit_trajectory(name):
    """oracle generate(basic_unit=u) == the reference's generate, bit for bit: final mask and pattern, every log line,
    numpy and torch RNG positions (u = 1: per-pixel groups, many of them all-zero; 4: groups straddling the 7-px density
    windows; 14: groups larger than a density window)."""
    tiny = MG.TinyNet().eval()
    x = torch.from_numpy(GB["bu_x"])
    assert torch.equal(x, MBU.image())
    kw = MBU.run_kwargs(name, tiny, x)
    _seed()
    log = []
    m, p = OA.generate(tiny, x, n_classes=1000, log=log.append, **kw)
    gm = GB["bu_%s_mask" % name]
    if gm.dtype == np.uint8:
        assert np.array_equal(np.packbits(m.numpy().astype(bool)), gm)
    else:
        assert np.array_equal(m.numpy(), gm)
    assert np.array_equal(p.numpy(), GB["bu_%s_pattern" % name])
    assert log == [str(s) for s in GB["bu_%s_log" % name]]
    assert np.array_equal(np.random.get_state()[1][:4], GB["bu_%s_rng_np" % name])
    assert np.array_equal(torch.rand(3).numpy(), GB["bu_%s_rng_t" % name])


@pytest.mark.parametrize("size,unit", [(56, 0), (56, 3), (56, 5), (56, 57), (56, -7), (56, 3.5), (56, True), (224, 6)])
def test_invalid_basic_unit_raises_before_any_rng_draw(size, unit):
    """A basic_unit that is not a positive integer dividing the image size raises ValueError before the torch or numpy
    RNG moves (and before a device is needed); the reference would fail later, at stage 1's clip broadcast."""
    from dorpatch_b200.attack import DorPatch
    x = torch.rand(1, 3, size, size)
    _seed(7)
    t0, n0 = torch.get_rng_state(), np.random.get_state()
    with pytest.raises(ValueError, match="basic_unit"):
        DorPatch().generate(None, x, 0.1, 1000, "results/a/b", 0, basic_unit=unit)
    n1 = np.random.get_state()
    assert torch.equal(torch.get_rng_state(), t0) and np.array_equal(n0[1], n1[1]) and n0[2] == n1[2]


def test_basic_unit_is_part_of_the_result_path(tmp_path, monkeypatch):
    """--basic_unit N changes the patches and the stage-0 mask, so a non-default unit gets its own directory (stage-0
    cache included); the default path, and the order of the other suffixes, are unchanged."""
    from dorpatch_b200 import main as M
    from dorpatch_b200.utils import generate_saving_path
    monkeypatch.chdir(tmp_path)
    top = "results/dataset=imagenet_base_arch=resnetv2_targeted=False_attack=DorPatch_dropout=2_density=0.001_structured=0.001"
    sub = "/num_patch=-1_patch_budget=0.12"

    def path(argv):
        return generate_saving_path(vars(M.parser.parse_args(argv)).copy())

    assert M.parser.parse_args([]).basic_unit == 7
    assert path([]) == top + sub
    assert path(["--basic_unit", "7"]) == top + sub
    assert path(["--basic_unit", "14"]) == top + "__basic_unit=14" + sub
    assert path(["--attack_pc_n_patch", "2", "--synthetic", "2"]) == top + "__synthetic=2_attack_pc_n_patch=2" + sub
    assert path(["--basic_unit", "4", "--synthetic", "2", "--attack_pc_n_patch", "2"]) == \
        top + "__synthetic=2_attack_pc_n_patch=2_basic_unit=4" + sub
    for bad in ("3.5", "seven", ""):
        with pytest.raises(SystemExit):
            M.parser.parse_args(["--basic_unit", bad])
