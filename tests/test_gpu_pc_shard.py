"""PatchCleanser evaluation sharded over ranks, on the H100.

The claim the sharding rests on: forwarding a call's samples as chunk-aligned slices, one call per rank, gives the
labels and logits of the whole call bit for bit, at fp32, tf32 and bf16, at chunk 64 and 128, for the two-patch round 1
(630 samples) and certificate (22 680), at world 2, 3 and 8 -- and the launches of the slices add up to the call's.
Then robust_predict in a simulated world (ranks as threads sharing the one engine, their forwards in turn) returns the
single-process records, with the same launch count in total.  With two or more GPUs, torchrun of main.py on 2 GPUs
writes the PatchCleanser records and prints the metrics line of a single-process run, byte for byte."""
import contextlib
import glob
import importlib.util
import io
import os
import shutil
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from dorpatch_b200 import masks as PM
from dorpatch_b200.attack import shard_range

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
H = 112


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


SIM = _load("pc_shard_sim")


def _window(r, n_patch):
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow
    with contextlib.redirect_stdout(io.StringIO()):
        return MaskWindow(H, r, n_patch)


@pytest.fixture(scope="module")
def net():
    from dorpatch_b200.resnetv2 import ResNetV2
    torch.cuda.set_device(0)
    n = ResNetV2(seed=0)
    yield n
    for eng, _ in n._engines.values():
        eng.close()
    n._engines.clear()


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("chunk", [64, 128])
def test_chunk_aligned_slices_equal_the_whole_call(net, precision, chunk):
    eng = net.engine(H, precision=precision, chunk=chunk)
    mw = _window(0.12, 2)
    img = torch.rand(1, 3, H, H, generator=torch.Generator().manual_seed(11)).cuda()
    for table in (mw.mask_rects, mw.double_mask_rects):
        rects = PM.gather(table, np.arange(len(table)))
        n = len(rects)
        eng.predict(img, n, rects)                                          # every shape of this call warmed up
        c0 = eng.launch_count
        want_p, want_l = eng.predict(img, n, rects, return_logits=True)
        want_launches = eng.launch_count - c0
        for world in (2, 3, 8):
            ps, ls = [], []
            c0 = eng.launch_count
            for r in range(world):
                lo, hi = shard_range(n, r, world, chunk)
                if hi > lo:
                    p, lg = eng.predict(img, hi - lo, rects[lo:hi], return_logits=True)
                    ps.append(p)
                    ls.append(lg)
            got_p, got_l = np.concatenate(ps), np.concatenate(ls)
            assert np.array_equal(got_p, want_p), (n, world)
            assert got_l.tobytes() == want_l.tobytes(), (n, world, float(np.abs(got_l - want_l).max()))
            assert eng.launch_count - c0 == want_launches, (n, world)
        if n == 630:
            assert len(np.unique(want_p)) > 1                               # labels that can disagree, not a constant


def _simulated(net, mw, img, world):
    """robust_predict(img, True) on `world` simulated ranks sharing net's engine: (records per rank, launches)."""
    from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
    lock = threading.Lock()
    eng = net.engine(H)
    c0 = eng.launch_count

    def rank_fn(d):
        pc = PatchCleanser(mw, net)
        pc._group = lambda: d
        predict = pc._predict

        def locked(im, rects):
            with lock:
                return predict(im, rects)
        pc._predict = locked
        return pc.robust_predict(img, True), pc.forwards

    out = SIM.ThreadWorld(world).run(rank_fn)
    return [r for r, _ in out], [f for _, f in out], eng.launch_count - c0


def _images(net, mw):
    """A unanimous image (uniform 0.5: occluding it changes nothing) and the random image of the fewest minority samples
    in round 1 among a few -- one that takes the second round."""
    eng = net.engine(H)
    single = PM.gather(mw.mask_rects, np.arange(len(mw.mask_rects)))
    best = None
    for s in range(8):
        im = torch.rand(3, H, H, generator=torch.Generator().manual_seed(100 + s)).cuda()
        p = eng.predict(im[None], len(single), single)
        vals, counts = np.unique(p, return_counts=True)
        minority = len(p) - counts.max()
        if minority > 0 and (best is None or minority < best[0]):
            best = (minority, im)
    assert best is not None, "no candidate image takes the second round"
    return torch.full((3, H, H), 0.5, device="cuda"), best[1]


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
def test_robust_predict_in_a_simulated_world_equals_one_process(net, precision, monkeypatch):
    from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
    monkeypatch.setenv("DORPATCH_PRECISION", precision)
    mw = _window(0.12, 2)
    unanimous, split = _images(net, mw)
    eng = net.engine(H)
    rounds = []
    for img in (unanimous, split):
        PatchCleanser(mw, net).robust_predict(img, True)                    # warm-up: every call shape once
        pc = PatchCleanser(mw, net)
        c0 = eng.launch_count
        want = pc.robust_predict(img, True)
        want_launches = eng.launch_count - c0
        rounds.append(len(np.unique(want.preds_1)) > 1)
        for world in (2, 3):
            recs, forwards, launches = _simulated(net, mw, img, world)
            for r, rec in enumerate(recs):
                assert SIM.records_equal(rec, want), (precision, world, r)
            assert sum(forwards) == pc.forwards and launches == want_launches, (world, forwards, pc.forwards)
    assert rounds == [False, True]


def _run(cmd, env, cwd, timeout):
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, cwd=cwd, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("clean accuracy:")]
    assert len(lines) == 1, out.stdout[-3000:]
    return lines[0]


def test_torchrun_main_records_equal_one_process(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), DORPATCH_AUTOTUNE="0")
    env.pop("DORPATCH_SHARD", None)
    main = os.path.join(ROOT, "main.py")
    args = ["--synthetic", "2", "--random_init", "--max_iterations", "20", "--sampling_size", "16"]
    single = [sys.executable, main] + args
    dist = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
            "127.0.0.1", "--master-port", "29541", main] + args
    _run(single + ["--pc_n_patch", "1"], env, tmp_path, 3600)             # generates the patches (and one-patch records)
    for n_patch, name in ((2, "adv_PC2_*.pt"), (1, "adv_PC_*.pt")):
        files = lambda: sorted(glob.glob(os.path.join(str(tmp_path), "results", "**", name), recursive=True))
        for f in files():
            os.remove(f)
        line_1 = _run(single + ["--pc_n_patch", str(n_patch)], env, tmp_path, 3600)
        want = {f: open(f, "rb").read() for f in files()}
        assert len(want) == 2, want.keys()
        for f in want:
            os.remove(f)
        line_2 = _run(dist + ["--pc_n_patch", str(n_patch)], env, tmp_path, 3600)
        got = {f: open(f, "rb").read() for f in files()}
        assert line_2 == line_1, (line_1, line_2)
        assert got == want, [os.path.basename(f) for f in want if got.get(f) != want[f]]
    shutil.rmtree(os.path.join(str(tmp_path), "results"), ignore_errors=True)
