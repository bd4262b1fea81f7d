"""Generation against the two-patch PatchCleanser window on the GPU: device failed-mask bitmaps sized for the 90 720-mask
universe, the deduplicated universe scan against a full dp_predict, generate with device and host failed sets, generate
against the oracle, and the main.py driver with --attack_pc_n_patch 2."""
import contextlib
import io
import os
import random

import numpy as np
import pytest
import torch

from dorpatch_b200 import masks as PM
from oracle import resnetv2 as OR, two_patch_attack as OTA

pytestmark = pytest.mark.gpu
N_MASK = 90720
RATIOS = len(PM.DROPOUT_SIZES)


def _seed(s=1234):
    random.seed(s)
    torch.manual_seed(s)
    np.random.seed(s)


def test_device_failed_set_over_two_patch_universe_equals_host(oracle_params):
    """dp_failed_set_reset(90 720) then write / update / read against the host list arithmetic of attack.py:259-267
    (_ImageState.bookkeeping with n_failed=None) over 400 random steps of two images, indices up to 90 719.  An engine
    that never called dp_failed_set_reset keeps its 4096-mask capacity."""
    from dorpatch_b200.attack import _ImageState
    from dorpatch_b200.engine import Engine
    e = Engine(img=56, precision="fp32", chunk=8, max_images=2, autotune=False)
    fresh = Engine(img=56, precision="fp32", chunk=8, max_images=2, autotune=False)
    try:
        e.failed_reset(N_MASK)
        B, S = 2, 16
        host = [_ImageState(0.01, 1e-3, 3, False, np.random.RandomState(10 + b)) for b in range(B)]
        dev = [_ImageState(0.01, 1e-3, 3, False, np.random.RandomState(10 + b)) for b in range(B)]
        for b, s in enumerate(dev):
            s.dev = (e, b)
        rng = np.random.RandomState(0)
        for b in range(B):
            init = sorted(set(rng.choice(N_MASK, 40, replace=False).tolist()) | {0, 4096, N_MASK - 1})
            host[b].failed, host[b].n_failed = list(init), len(init)
            dev[b].set_failed(init)
        top = 0
        for i in range(990, 1390):                   # crosses i == 1000, where half of the samples start to come from the set
            idx_h, idx_d, nff_h, nff_d = [], [], [], []
            for b in range(B):
                a, na = host[b].sample(i, N_MASK, S)
                c, nc = dev[b].sample(i, N_MASK, S)
                assert na == nc and np.array_equal(a, c)
                idx_h.append(a); nff_h.append(na); idx_d.append(c); nff_d.append(nc)
                top = max(top, int(c.max()))
            loss = (rng.rand(B, S) < 0.6).astype(np.float32) * 0.5
            counts = e.failed_update(np.stack(idx_d), nff_d, [True] * B, loss=loss)
            for b in range(B):
                ra = host[b].bookkeeping(1, i, loss[b], idx_h[b], nff_h[b], 1.0)
                rb = dev[b].bookkeeping(1, i, loss[b], idx_d[b], nff_d[b], 1.0, n_failed=counts[b])
                assert ra == rb and host[b].n_failed == dev[b].n_failed == counts[b]
            if i % 50 == 0:
                for b in range(B):
                    assert e.failed_read(b) == host[b].failed
        assert top > 4096 * 16
        with pytest.raises(RuntimeError):
            e.failed_write(0, [N_MASK])
        e.failed_reset(N_MASK)                       # clears every image's set
        assert e.failed_read(0) == [] and e.failed_read(1) == []

        fresh.failed_write(0, [0, 4095])
        assert fresh.failed_read(0) == [0, 4095]
        with pytest.raises(RuntimeError):
            fresh.failed_write(0, [4096])
        with pytest.raises(RuntimeError):
            fresh.failed_update(np.full((1, 1), 4096, np.int32), [0], [True], loss=np.ones((1, 1), np.float32))
    finally:
        e.close()
        fresh.close()


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
def test_distinct_scan_equals_full_predict(engine_factory, precision):
    """dp_predict over the 31 080 distinct occlusions, spread through inv, against dp_predict over all 90 720 masks, for
    two 56 px images.  fp32: equal on every mask.  tf32 / bf16: a sample's logits can change in the last bits with the
    batch it is computed in (measured: 2-14 labels of 90 720 differ), so a label may flip where the full scan's top
    logit and the distinct scan's label are within that noise: at most 0.1 % of the masks, each a near-tie in the full
    scan's own logits (margin <= 1 % of the row's logit range)."""
    e = engine_factory(img=56, precision=precision, chunk=256, max_images=1)
    t = PM.universe(56, 2, 2)
    distinct, inv = PM.distinct_occlusions(t, RATIOS)
    full_rects, few_rects = PM.gather(t, np.arange(len(t))), PM.gather(distinct, np.arange(len(distinct)))
    for seed in (3, 4):
        img = torch.rand(1, 3, 56, 56, generator=torch.Generator().manual_seed(seed)).cuda()
        full, logits = e.predict(img, len(t), full_rects, return_logits=True)
        few = e.predict(img, len(distinct), few_rects)[inv]
        off = np.nonzero(full != few)[0]
        margin = logits[off, full[off]] - logits[off, few[off]]
        spread = logits[off].max(1) - logits[off].min(1)
        print(precision, "image", seed, "labels", len(np.unique(full)), "masks off", len(off),
              "max margin / range", float((margin / spread).max()) if len(off) else 0.0)
        if precision == "fp32":
            assert len(off) == 0
        assert len(off) <= len(t) // 1000
        assert (margin <= 0.01 * spread).all()


@pytest.fixture(scope="module")
def native_model(oracle_params):
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    saved = {k: os.environ.get(k) for k in ("DORPATCH_PRECISION", "DORPATCH_CHUNK")}
    os.environ["DORPATCH_PRECISION"], os.environ["DORPATCH_CHUNK"] = "fp32", "64"
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    yield torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _generate(model, x, save_dir, **kw):
    from dorpatch_b200.attack import DorPatch
    _seed()
    buf = io.StringIO()
    atk = DorPatch()
    with contextlib.redirect_stdout(buf):
        m, p = atk.generate(model, x.cuda(), save_dir=save_dir, batch_id=0, **kw)
    log = [l for l in buf.getvalue().splitlines() if not l.startswith("mask size")]
    return m.cpu(), p.cpu(), log, np.random.get_state()[1][:4].copy(), atk.last_stats


def test_generate_two_patch_dropout2_device_sets_equal_host_sets(native_model, tmp_path, monkeypatch):
    """generate(pc_n_patch=2, dropout=2) at fp32, 56 px, S=16, 150 iterations per stage (scans at i = 0 and 100): the
    failed sets as device bitmaps over the 90 720-mask universe and as host lists give the identical run -- mask,
    pattern, every log line, numpy RNG position.  Every scan forwards the 31 080 distinct occlusions."""
    x = torch.rand(1, 3, 56, 56, generator=torch.Generator().manual_seed(21))
    kw = dict(patch_budget=0.12, n_classes=1000, targeted=True, y=torch.tensor([7]).cuda(), max_iterations=150,
              sampling_size=16, dropout=2, pc_n_patch=2)
    dev = _generate(native_model, x, str(tmp_path / "dev" / "sub"), **kw)
    monkeypatch.setenv("DORPATCH_FAILED", "host")
    host = _generate(native_model, x, str(tmp_path / "host" / "sub"), **kw)
    assert torch.equal(dev[0], host[0]) and torch.equal(dev[1], host[1])
    assert dev[2] == host[2] and np.array_equal(dev[3], host[3])
    for stats in (dev[4], host[4]):
        assert stats["scans"] == 4 and stats["scan_forwards"] == 4 * 31080, stats
    assert sum(l.startswith(">> ") for l in dev[2]) == 4


def test_generate_two_patch_dropout1_matches_oracle(native_model, oracle_params, tmp_path):
    """generate(pc_n_patch=2, dropout=1) at fp32, 112 px, targeted, 2 stages x 3 iterations, against the oracle on
    the same seeds, S=8: identical numpy RNG consumption and log structure, patch mask IoU >= 0.90, at most 5 % of the
    pattern's pixels off by more than lr/4 (sign(grad) steps of last-bit gradient differences, as in
    test_gpu_generate._compare)."""
    H, LR = 112, 0.01
    x = torch.rand(1, 3, H, H, generator=torch.Generator().manual_seed(7))
    kw = dict(patch_budget=0.12, n_classes=1000, targeted=True, max_iterations=3, sampling_size=8, dropout=1, lr=LR)
    tgt = torch.tensor([321])
    m_gpu, p_gpu, log_gpu, rng_gpu, stats = _generate(native_model, x, str(tmp_path / "c" / "sub"), y=tgt.cuda(),
                                                      pc_n_patch=2, **kw)
    assert stats["scan_forwards"] == stats["scans"] * 2520
    net = OR.OracleNet(oracle_params, weights_require_grad=False).eval()
    _seed()
    log_or = []
    m_or, p_or = OTA.generate(net, x, y=tgt, log=log_or.append, pc_n_patch=2, **kw)
    rng_or = np.random.get_state()[1][:4].copy()
    assert np.array_equal(rng_gpu, rng_or)
    assert len(log_gpu) == len(log_or)
    for a, b in zip(log_gpu, log_or):
        print("GPU:", a)
        print("ORA:", b)
        assert a.split(",")[0] == b.split(",")[0]
    inter = ((m_gpu > 0.5) & (m_or > 0.5)).sum().item()
    union = ((m_gpu > 0.5) | (m_or > 0.5)).sum().item()
    iou = inter / max(union, 1)
    frac = ((p_gpu - p_or).abs() > 0.25 * LR).float().mean().item()
    print("mask IoU", iou, "pattern pixels off by > lr/4", frac)
    assert iou >= 0.90 and frac <= 0.05, (iou, frac)


def test_main_driver_attack_two_patch(tmp_path, monkeypatch):
    """main.py --attack_pc_n_patch 2 --pc_n_patch 2 end to end: patches and records under the `__attack_pc_n_patch=2`
    directory, the stage-0 cache in its parent; a later default run in the same root uses its own directory and neither
    reads nor overwrites the two-patch artefacts."""
    from dorpatch_b200 import main as M
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("DORPATCH_PRECISION", "bf16")
    base = ["--synthetic", "2", "--random_init", "--img_size", "56", "--max_iterations", "150", "--sampling_size", "16"]

    def run(extra):
        with contextlib.redirect_stdout(io.StringIO()):
            return M.cli(base + extra)

    two = run(["--attack_pc_n_patch", "2", "--pc_n_patch", "2"])
    rd = two["result_dir"]
    assert rd.split(os.sep)[1].endswith("_attack_pc_n_patch=2") and rd.endswith("num_patch=-1_patch_budget=0.12")
    assert two["line"].startswith("clean accuracy: ") and len(two["acc_PC"]) == 4
    stored = [os.path.join(rd, f % i) for i in range(2) for f in ("adv_mask_%d.pt", "adv_pattern_%d.pt", "adv_PC2_%d.pt")]
    stored += [os.path.join(os.path.dirname(rd), f % i) for i in range(2) for f in ("adv_mask_%d.pt", "adv_pattern_%d.pt")]
    for f in stored:
        assert os.path.exists(f), f
    mtimes = {f: os.stat(f).st_mtime_ns for f in stored}

    one = run([])
    assert one["result_dir"] != rd and "attack_pc_n_patch" not in one["result_dir"]
    assert os.path.dirname(one["result_dir"]) != os.path.dirname(rd)
    for i in range(2):
        assert os.path.exists(os.path.join(one["result_dir"], "adv_PC_%d.pt" % i))
    assert {f: os.stat(f).st_mtime_ns for f in stored} == mtimes
    assert sorted(os.listdir(rd)) == sorted(os.path.basename(f) for f in stored[:6])
