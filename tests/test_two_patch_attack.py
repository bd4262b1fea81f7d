"""Generation against the two-patch PatchCleanser window (DorPatch.generate(pc_n_patch=2)), on the CPU: the oracle
against the reference's trajectories, the two-patch universe against the reference's tables, the distinct-occlusion
map of the universe scans, their sharding over a world-2 gloo group, argument checks and the result path."""
import importlib.util
import os
import random
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from dorpatch_b200 import masks as PM
from oracle import attack as OA, two_patch_attack as OTA

HERE = os.path.dirname(os.path.abspath(__file__))
RATIOS = (0.015, 0.03, 0.06, 0.12)


def _module(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, "golden", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MG = _module("make_golden")
MTA = _module("make_two_patch_attack_golden")
GA = MTA.load()
GT = _module("make_two_patch_golden").load()


def _seed(s=1234):
    random.seed(s)
    torch.manual_seed(s)
    np.random.seed(s)


@pytest.mark.parametrize("name", list(MTA.RUNS))
def test_oracle_reproduces_reference_two_patch_trajectory(name):
    """oracle generate(pc_n_patch=2) == the reference's generate over MaskWindow(56, r, 2), bit for bit: final mask and
    pattern, every log line, numpy and torch RNG positions.  d2 samples from a non-empty failed set at i >= 1000."""
    tiny = MG.TinyNet().eval()
    x = torch.from_numpy(GA["tpa_x"])
    assert torch.equal(x, MTA.image())
    kw = MTA.run_kwargs(name, tiny, x)
    _seed()
    log = []
    m, p = OTA.generate(tiny, x, n_classes=1000, pc_n_patch=2, log=log.append, **kw)
    gm = GA["tpa_%s_mask" % name]
    if gm.dtype == np.uint8:
        assert np.array_equal(np.packbits(m.numpy().astype(bool)), gm)
    else:
        assert np.array_equal(m.numpy(), gm)
    assert np.array_equal(p.numpy(), GA["tpa_%s_pattern" % name])
    assert log == [str(s) for s in GA["tpa_%s_log" % name]]
    assert np.array_equal(np.random.get_state()[1][:4], GA["tpa_%s_rng_np" % name])
    assert np.array_equal(torch.rand(3).numpy(), GA["tpa_%s_rng_t" % name])
    if name == "d2":
        assert any(n > 0 for n in MTA.failed_at_1000(log))


@pytest.mark.parametrize("dropout", [1, 2])
def test_two_patch_universe_is_the_references(dropout):
    """masks.universe(56, d, 2): 2 520 / 90 720 masks, ratio-major, each ratio's block in the reference's order
    (pairs: packed bits; triples: occluded-pixel count of every mask and the probe masks)."""
    H = 56
    t = PM.universe(H, dropout, 2)
    n = 630 if dropout == 1 else 22680
    assert t.shape == (4 * n, 2 if dropout == 1 else 3, 4)
    for q, r in enumerate(RATIOS):
        keep = PM.to_bool(t[q * n:(q + 1) * n], H)
        if dropout == 1:
            assert np.array_equal(np.packbits(keep), GT["tp_single_%d_%s" % (H, r)])
        else:
            assert np.array_equal((~keep).reshape(n, -1).sum(1), GT["tp_double_sum_%d_%s" % (H, r)])
            assert np.array_equal(np.packbits(keep[list(GT["tp_probes"])]), GT["tp_double_probe_%d_%s" % (H, r)])


@pytest.mark.parametrize("n_patch,dropout", [(1, 1), (1, 2), (2, 1), (2, 2)])
def test_distinct_occlusion_map_is_exact(n_patch, dropout):
    """distinct[inv[k]] occludes exactly the pixels table[k] does, for every k.  The two-patch dropout-2 universe has
    7 770 distinct occlusions per ratio; every other universe maps to itself."""
    H = 56
    t = PM.universe(H, dropout, n_patch)
    distinct, inv = PM.distinct_occlusions(t, len(RATIOS))
    assert inv.shape == (len(t),) and inv.min() == 0 and inv.max() == len(distinct) - 1
    n = len(t) // len(RATIOS)
    for q in range(len(RATIOS)):
        block = slice(q * n, (q + 1) * n)
        assert np.array_equal(PM.to_bool(distinct[inv[block]], H), PM.to_bool(t[block], H))
        if n_patch == 2 and dropout == 2:
            assert len(np.unique(inv[block])) == 7770
    if n_patch == 2 and dropout == 2:
        assert len(distinct) == 31080
        first = np.unique(inv, return_index=True)[1]                # distinct[j] is the first mask of its class, in order
        assert (np.diff(first) > 0).all() and np.array_equal(distinct, t[first])
    else:
        assert np.array_equal(distinct, t) and np.array_equal(inv, np.arange(len(t)))


def test_oracle_scan_over_distinct_occlusions_equals_full_scan():
    """collect_failure over the 31 080 distinct occlusions, expanded through inv, == collect_failure over all 90 720
    masks of the two-patch dropout-2 universe (TinyNet, an image near a decision boundary)."""
    H = 56
    tiny = MG.TinyNet().eval()
    img = _module("make_two_patch_golden").two_patch_image(1158)[None]
    with torch.no_grad():
        y = int(tiny(img).argmax(-1))
    t = PM.universe(H, 2, 2)
    distinct, inv = PM.distinct_occlusions(t, len(RATIOS))
    full = OA.collect_failure(tiny, img, y, torch.from_numpy(PM.to_bool(t, H)), False, 1024)
    few = OA.collect_failure(tiny, img, y, torch.from_numpy(PM.to_bool(distinct, H)), False, 1024)
    f = np.zeros(len(distinct), bool)
    f[few] = True
    assert 0 < len(full) < len(t)
    assert np.nonzero(f[inv])[0].tolist() == full


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fake_predict(rects):
    """A label that depends only on the set of rectangles a sample occludes."""
    r = rects.astype(np.int64)
    key = np.sort((r[..., 0] << 48) | (r[..., 1] << 32) | (r[..., 2] << 16) | r[..., 3], axis=1)
    key[:, 1:][key[:, 1:] == key[:, :-1]] = 0
    return ((key % 1000003).sum(1) % 5).astype(np.int32)


def _scan_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dorpatch_b200.attack import scan_failures
    t = PM.universe(56, 2, 2)
    distinct, inv = PM.distinct_occlusions(t, len(RATIOS))
    full = PM.gather(t, np.arange(len(t)))
    rects = PM.gather(distinct, np.arange(len(distinct)))
    ok = True
    for y, targeted in ((3, False), (1, True)):
        seen = []

        def predict(r):
            seen.append(r.copy())
            return _fake_predict(r)

        want = scan_failures(_fake_predict, full, y, targeted)
        got = scan_failures(predict, rects, y, targeted, dist, "cpu", inv=inv)
        per = -(-len(rects) // world)
        mine = rects[rank * per:(rank + 1) * per]
        ok = ok and 0 < len(want) < len(t) and got == want and np.array_equal(np.concatenate(seen), mine)
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_distinct_scan_is_sharded_over_ranks_world2():
    """Under torch.distributed each rank forwards its contiguous shard of the distinct occlusions, and every rank ends
    with the sorted universe indices a full single-process scan returns."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_scan_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]


@pytest.mark.parametrize("kw", [dict(dual=True, dropout=2, pc_n_patch=2), dict(pc_n_patch=3), dict(pc_n_patch=0)])
def test_unsupported_configurations_raise_before_any_rng_draw(kw):
    """dual=True with the two-patch dropout-2 universe (6 rectangles per sample) and pc_n_patch outside {1, 2} raise
    NotImplementedError before the torch or numpy RNG moves (and before a device is needed)."""
    from dorpatch_b200.attack import DorPatch
    x = torch.rand(1, 3, 56, 56)
    _seed(7)
    t0, n0 = torch.get_rng_state(), np.random.get_state()
    with pytest.raises(NotImplementedError):
        DorPatch().generate(None, x, 0.1, 1000, "results/a/b", 0, **kw)
    n1 = np.random.get_state()
    assert torch.equal(torch.get_rng_state(), t0) and np.array_equal(n0[1], n1[1]) and n0[2] == n1[2]


def test_attack_pc_n_patch_is_part_of_the_result_path(tmp_path, monkeypatch):
    """--attack_pc_n_patch 2 changes the patches, so its results (and the stage-0 cache in the parent directory) get
    their own directory; the default path is unchanged, and --pc_n_patch (evaluation only) still changes nothing."""
    from dorpatch_b200 import main as M
    from dorpatch_b200.utils import generate_saving_path
    monkeypatch.chdir(tmp_path)
    top = "results/dataset=imagenet_base_arch=resnetv2_targeted=False_attack=DorPatch_dropout=2_density=0.001_structured=0.001"
    sub = "/num_patch=-1_patch_budget=0.12"

    def path(argv):
        return generate_saving_path(vars(M.parser.parse_args(argv)).copy())

    assert M.parser.parse_args([]).attack_pc_n_patch == 1
    assert path([]) == top + sub
    assert path(["--pc_n_patch", "2"]) == top + sub
    assert path(["--attack_pc_n_patch", "1"]) == top + sub
    assert path(["--attack_pc_n_patch", "2"]) == top + "__attack_pc_n_patch=2" + sub
    assert path(["--attack_pc_n_patch", "2", "--pc_n_patch", "2"]) == top + "__attack_pc_n_patch=2" + sub
    assert path(["--attack_pc_n_patch", "2", "--synthetic", "2"]) == top + "__synthetic=2_attack_pc_n_patch=2" + sub
    with pytest.raises(SystemExit):
        M.parser.parse_args(["--attack_pc_n_patch", "3"])
