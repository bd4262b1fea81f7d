"""Resumable DorPatch.generate on the GPU: a run cut at chosen steps and resumed from its checkpoint returns, prints,
counts and leaves the RNG streams exactly as one uninterrupted run.  fp32 engine and DORPATCH_AUTOTUNE=0, so that every
engine picks the same library algorithms; tf32 and bf16 once each.

A cut is an exception raised by a wrapper of Engine.attack_grad at the step (stage, i) it is given; the next call with
the same arguments continues from the checkpoint file.  The log of the chain is, for every cut run, the lines it printed
up to its last checkpoint write, then everything the last run printed."""
import contextlib
import io
import os
import pickle
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from dorpatch_b200 import attack as A
from dorpatch_b200.engine import Engine

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ENV = dict(DORPATCH_PRECISION="fp32", DORPATCH_CHUNK="16", DORPATCH_AUTOTUNE="0")


class _Cut(Exception):
    """Raised in place of a step: the process 'dies' there."""


def _close_new_engines(before, nets=()):
    from dorpatch_b200 import runtime
    for e in [e for e in runtime._ENGINES if all(e is not o for o in before)]:
        e.close()
    for net in nets:
        for ent in net._engines.values():
            ent[0].close()


@pytest.fixture(scope="module")
def native_model(oracle_params):
    """fp32, chunk 16, no autotuning.  At teardown the environment is restored and every engine created meanwhile is
    closed, so later modules find the device memory free."""
    from dorpatch_b200 import runtime
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    saved = {k: os.environ.get(k) for k in ENV}
    os.environ.update(ENV)
    before = list(runtime._ENGINES)
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    yield torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()
    _close_new_engines(before, [net])
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _seed():
    random.seed(1234)
    torch.manual_seed(1234)
    np.random.seed(1234)


def _position(path):
    """(stage, i) of the step a run resumed from `path` starts with; (0, 0) without a file."""
    if path is None or not os.path.exists(path):
        return 0, 0
    ck = torch.load(path, weights_only=True)
    return int(ck["stage"]), int(ck["i"])


def _cut_at(mp, cut, start):
    """Make Engine.attack_grad raise _Cut at step `cut` = (stage, i) of a run that starts at step `start`."""
    grad = Engine.attack_grad
    calls = [0, 0]

    def attack_grad(self, *a, **k):
        stage = int(a[8])
        i = (start[1] if stage == start[0] else 0) + calls[stage]
        calls[stage] += 1
        if (stage, i) == cut:
            raise _Cut()
        return grad(self, *a, **k)

    mp.setattr(Engine, "attack_grad", attack_grad)


def _run(monkeypatch, model, x, kw, ckpt=None, every=100, cut=None, save_dir=None, hook=None):
    """One generate() call from a freshly seeded process state; returns what it returned, printed, counted and left."""
    _seed()
    buf = io.StringIO()
    out = dict(cut=False, lines_at_ckpt=0, start=_position(ckpt))
    with monkeypatch.context() as mp:
        save = A.save_checkpoint

        def counted_save(path, ck):
            if ckpt is None:
                raise AssertionError("checkpoint=None wrote a checkpoint")
            save(path, ck)
            out["lines_at_ckpt"] = len(buf.getvalue().splitlines())

        mp.setattr(A, "save_checkpoint", counted_save)
        if cut is not None:
            _cut_at(mp, cut, out["start"])
        if hook is not None:
            hook(mp)
        with contextlib.redirect_stdout(buf):
            try:
                gen = A.DorPatch()
                out["m"], out["p"] = gen.generate(model, x, 0.12, 1000, save_dir, 0, checkpoint=ckpt,
                                                  checkpoint_every=every, **kw)
                out["stats"] = gen.last_stats
            except _Cut:
                out["cut"] = True
    out["log"] = buf.getvalue().splitlines()
    out["np"], out["torch"] = np.random.get_state(), torch.get_rng_state()
    return out


def _assert_same(a, b):
    assert torch.equal(a["m"], b["m"]) and torch.equal(a["p"], b["p"])
    assert a["log"] == b["log"]
    assert a["stats"] == b["stats"]
    assert a["np"][0] == b["np"][0] and np.array_equal(a["np"][1], b["np"][1]) and a["np"][2:] == b["np"][2:]
    assert torch.equal(a["torch"], b["torch"])


def _chain(monkeypatch, model, x, kw, tmp_path, every, cuts, want_positions, save_dir=None, hook=None, check=None):
    """Cut at every step of `cuts` in turn, each run resuming from the last one's checkpoint; check the checkpoint's
    position after each cut, then finish.  Returns the chain's combined result (log stitched as the module says)."""
    ckpt = str(tmp_path / "adv_ckpt_0.pt")
    log = []
    for k, (cut, want) in enumerate(zip(cuts, want_positions)):
        r = _run(monkeypatch, model, x, kw, ckpt, every, cut, save_dir, hook)
        assert r["cut"], "the run ended before step %s" % (cut,)
        assert _position(ckpt) == want, (cut, _position(ckpt))
        if check is not None:
            check(k, r, torch.load(ckpt, weights_only=True))
        log += r["log"][:r["lines_at_ckpt"]]
    r = _run(monkeypatch, model, x, kw, ckpt, every, None, save_dir, hook)
    assert not r["cut"]
    assert not os.path.exists(ckpt), "a successful return deletes the checkpoint"
    r["log"] = log + r["log"]
    return r


def _image(B=1, seed=7):
    return torch.rand(B, 3, 112, 112, generator=torch.Generator().manual_seed(seed)).cuda()


def test_host_sampler_cuts_at_the_switch_the_failed_set_the_boundary_and_stage1(native_model, monkeypatch, tmp_path):
    """B = 1, untargeted, the global numpy stream.  Cuts: before step 500; exactly at 500, so the resumed run switches to
    targeted from the saved adv_x_prev / last_preds; after 1000, so it samples from a restored failed set; at stage 1's
    first step, right after the stage-boundary checkpoint; inside stage 1.  Stage 0's end-of-stage work (the stage-0
    save) runs once in the whole chain.  The uninterrupted run uses checkpoint=None and writes nothing.
    Early stops are switched off here (bookkeeping's stop flag forced to False, in every run alike), so that both stages
    run all 1100 steps and every cut lands where it is placed; test_stopped_image_stays_stopped covers stops."""
    x = _image()
    kw = dict(max_iterations=1100, sampling_size=8, dropout=1)
    stage0_saves = []
    save = torch.save

    def hook(mp):
        bk = A._ImageState.bookkeeping
        mp.setattr(A._ImageState, "bookkeeping", lambda self, *a, **k: (bk(self, *a, **k)[0], False))

        def counting_save(obj, f, *a, **k):
            if isinstance(f, str) and f.endswith("adv_mask_0.pt"):
                stage0_saves.append(f)
            return save(obj, f, *a, **k)
        mp.setattr(torch, "save", counting_save)

    ref_dir, dir0 = tmp_path / "ref", tmp_path / "chain"
    ref = _run(monkeypatch, native_model, x, kw, save_dir=str(ref_dir / "sub"), hook=hook)
    assert sorted(os.listdir(str(ref_dir))) == ["adv_mask_0.pt", "adv_pattern_0.pt"]   # the stage-0 save, nothing else
    assert ref["stats"]["steps"] == 2200
    del stage0_saves[:]
    (tmp_path / "run").mkdir()
    got = _chain(monkeypatch, native_model, x, kw, tmp_path / "run", 50,
                 cuts=[(0, 480), (0, 500), (0, 1030), (1, 0), (1, 730)],
                 want_positions=[(0, 450), (0, 500), (0, 1000), (1, 0), (1, 700)],
                 save_dir=str(dir0 / "sub"), hook=hook)
    _assert_same(ref, got)
    assert len(stage0_saves) == 1
    assert torch.equal(torch.load(str(ref_dir / "adv_mask_0.pt")), torch.load(str(dir0 / "adv_mask_0.pt")))


def test_device_sampler_dual_batch_of_four(native_model, monkeypatch, tmp_path):
    x = _image(4, seed=8)
    kw = dict(max_iterations=240, sampling_size=8, dropout=1, dual=True, eot_sampler="device",
              image_seeds=[11, 12, 13, 14])
    ref = _run(monkeypatch, native_model, x, kw)
    got = _chain(monkeypatch, native_model, x, kw, tmp_path, 40, cuts=[(0, 130), (1, 90)],
                 want_positions=[(0, 120), (1, 80)])
    _assert_same(ref, got)


def test_two_patch_universe(native_model, monkeypatch, tmp_path):
    x = _image(seed=9)
    kw = dict(max_iterations=150, sampling_size=8, dropout=1, pc_n_patch=2)
    ref = _run(monkeypatch, native_model, x, kw)
    got = _chain(monkeypatch, native_model, x, kw, tmp_path, 30, cuts=[(0, 100), (1, 45)],
                 want_positions=[(0, 90), (1, 30)])
    _assert_same(ref, got)


def test_stopped_image_stays_stopped(native_model, monkeypatch, tmp_path):
    """B = 2.  Image 0 stops at step 60 of stage 0 and image 1 at step 170 (forced through the stop flag that
    bookkeeping returns; everything a stop does follows from it).  The first cut, at 150, finds image 0 stopped: the
    resumed run keeps it inactive and keeps its best snapshot.  Image 1's stop then ends stage 0 early, so the
    stage-boundary checkpoint carries the stale gradient that stage 1's first update adds."""
    x = _image(2, seed=10)
    kw = dict(max_iterations=200, sampling_size=8, dropout=1, image_seeds=[5, 6])
    stops = {(0, 60, 0), (0, 170, 1)}
    seen = []

    def hook(mp):
        bk = A._ImageState.bookkeeping

        def bookkeeping(self, stage, i, *a, **k):
            seen.append((stage, i, self.dev[1]))
            improved, stop = bk(self, stage, i, *a, **k)
            return improved, stop or (stage, i, self.dev[1]) in stops
        mp.setattr(A._ImageState, "bookkeeping", bookkeeping)

    ref = _run(monkeypatch, native_model, x, kw, hook=hook)
    assert [l for l in ref["log"] if l.startswith("early stop")] == ["early stop at iteration:   60",
                                                                     "early stop at iteration:  170"]

    def check(k, r, ck):
        if k == 0:
            assert [d["active"] for d in ck["state"]["images"]] == [False, True]   # image 0 had stopped
            assert any(l == "early stop at iteration:   60" for l in r["log"])
            assert ck["state"]["have_stale"] and ck["state"]["stale_gp"] is not None
            del seen[:]
        else:
            assert not any(s == 0 and i >= 150 and b == 0 for s, i, b in seen)   # never book-kept again in stage 0
            assert ck["state"]["have_stale"]

    got = _chain(monkeypatch, native_model, x, kw, tmp_path, 25, cuts=[(0, 150), (1, 5)],
                 want_positions=[(0, 150), (1, 0)], hook=hook, check=check)
    _assert_same(ref, got)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_tf32_and_bf16(native_model, monkeypatch, tmp_path, precision):
    monkeypatch.setenv("DORPATCH_PRECISION", precision)
    x = _image(seed=12)
    kw = dict(max_iterations=120, sampling_size=8, dropout=1)
    ref = _run(monkeypatch, native_model, x, kw)
    got = _chain(monkeypatch, native_model, x, kw, tmp_path, 20, cuts=[(0, 70), (1, 50)],
                 want_positions=[(0, 60), (1, 40)])
    _assert_same(ref, got)


def _child(tmp_path, name, ckpt=None, cut=None):
    out = str(tmp_path / (name + ".pkl"))
    cmd = [sys.executable, os.path.join(HERE, "checkpoint_child.py"), out]
    if ckpt:
        cmd += ["--checkpoint", ckpt, "--every", "20"]
    if cut:
        cmd += ["--cut", "%d,%d" % cut]
    env = dict(os.environ, PYTHONPATH=ROOT, **ENV)
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
    with open(out, "rb") as f:
        return p.returncode, p.stdout.decode(errors="replace"), pickle.load(f)


def test_fresh_process_resume(tmp_path):
    """The interrupted run, the resumed run and the uninterrupted run are three processes; the interrupted one leaves
    through SystemExit at its cut."""
    ckpt = str(tmp_path / "adv_ckpt_0.pt")
    code, text, ref = _child(tmp_path, "ref")
    assert code == 0, text
    code, text, cut = _child(tmp_path, "cut", ckpt, (0, 70))
    assert code == 3 and cut["cut"], text
    assert _position(ckpt) == (0, 60)
    code, text, res = _child(tmp_path, "resumed", ckpt)
    assert code == 0, text
    assert not os.path.exists(ckpt)
    res["log"] = cut["log"][:cut["lines_at_ckpt"]] + res["log"]
    for k in ("m", "p"):
        assert torch.equal(ref[k], res[k])
    assert ref["log"] == res["log"] and ref["stats"] == res["stats"]
    assert ref["np"][0] == res["np"][0] and np.array_equal(ref["np"][1], res["np"][1]) and ref["np"][2:] == res["np"][2:]
    assert torch.equal(ref["torch"], res["torch"])


def test_main_resumes_an_interrupted_batch(tmp_path, monkeypatch):
    """main.py --checkpoint_every 50, cut in batch 0's stage 1 and rerun with the same flags: the same metrics line and
    the same artefacts, byte for byte, as one uninterrupted run."""
    from dorpatch_b200 import main as M
    from dorpatch_b200 import runtime
    monkeypatch.delenv("DORPATCH_PRECISION", raising=False)
    monkeypatch.delenv("DORPATCH_CHUNK", raising=False)
    monkeypatch.setenv("DORPATCH_AUTOTUNE", "0")
    argv = ["--synthetic", "2", "--random_init", "--max_iterations", "300", "--sampling_size", "8",
            "--checkpoint_every", "50"]

    def main(where, cut=None):
        (tmp_path / where).mkdir(exist_ok=True)
        before = list(runtime._ENGINES)
        with monkeypatch.context() as mp:
            mp.chdir(tmp_path / where)
            if cut is not None:
                _cut_at(mp, cut, (0, 0))                            # batch 0's generate() is the first call
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    return M.cli(argv)
            except _Cut:
                return None
            finally:
                _close_new_engines(before)

    ref = main("a")
    assert main("b", cut=(1, 120)) is None
    rd = os.path.join(str(tmp_path / "b"), ref["result_dir"])
    assert os.path.exists(os.path.join(rd, "adv_ckpt_0.pt")) and not os.path.exists(os.path.join(rd, "adv_mask_0.pt"))
    assert _position(os.path.join(rd, "adv_ckpt_0.pt")) == (1, 100)
    got = main("b")
    assert got["line"] == ref["line"]
    for i in range(2):
        for d, names in ((ref["result_dir"], ("adv_mask_%d.pt", "adv_pattern_%d.pt", "adv_PC_%d.pt")),
                         (os.path.dirname(ref["result_dir"]), ("adv_mask_%d.pt", "adv_pattern_%d.pt"))):
            for f in names:
                a = open(os.path.join(str(tmp_path / "a"), d, f % i), "rb").read()
                b = open(os.path.join(str(tmp_path / "b"), d, f % i), "rb").read()
                assert a == b, f % i
        assert not os.path.exists(os.path.join(str(tmp_path / "b"), ref["result_dir"], "adv_ckpt_%d.pt" % i))
