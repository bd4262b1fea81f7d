"""Step-level checkpoints of DorPatch.generate on the CPU: the per-image state and every RNG stream round-trip through a
checkpoint file, the refusals of a checkpoint written by another call, the atomic write, main.py's --checkpoint_every,
and the rank-0-writes / every-rank-reads protocol under a world-2 gloo group.  The resumed generate() itself runs on the
GPU (test_gpu_checkpoint.py)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from dorpatch_b200 import attack as A

KW = dict(patch_budget=0.12, targeted=False, lr=0.01, confidence=0.1, clip_min=0, clip_max=1, max_iterations=5000,
          basic_unit=7, selection="topk", dropout=2, sampling_size=128, density=1e-3, structured=1e-3, eps=4.0,
          dual=False, eot_affine=0.0, eot_colour=0.0, eot_seed=0, pc_n_patch=1, eot_sampler="host", image_seeds=None)


def _x():
    return torch.rand(2, 3, 56, 56, generator=torch.Generator().manual_seed(0))


def _fp(x=None, y=(3, 4), world=1, precision="fp32", **over):
    kw = dict(KW)
    kw.update(over)
    return A.checkpoint_fingerprint(_x() if x is None else x, list(y), world, precision, **kw)


def _ckpt(fp, **extra):
    ck = dict(version=A.CHECKPOINT_VERSION, fingerprint=fp, stage=0, i=100, state=dict(a=torch.arange(5)))
    ck.update(extra)
    return ck


def _draws(rs):
    return rs.choice(np.arange(2520), 16, replace=False), rs.randn(3), rs.rand(2)


def test_image_state_and_rng_streams_round_trip(tmp_path):
    path = str(tmp_path / "ck.pt")
    s = A._ImageState(0.01, 1e-3, 7, False, None)
    s.lr, s.loss_best, s.not_decay, s.num_failure = np.float32(0.001), np.float32(12.375), 57, 9
    s.coeff_group_lasso, s.structured = 1e-5 * A.SCALE_UP ** 3 / A.SCALE_DOWN, 1e-3 / A.SCALE_DOWN
    s.y, s.targeted, s.crit_targeted, s.certifiable, s.active = 42, True, True, False, False
    s.set_failed([3, 17, 2519])
    fresh = A._ImageState(0.01, 1e-3, 7, False, None)       # an untouched image: inf loss_best / num_failure, empty set

    np.random.seed(11)
    np.random.rand(5)
    torch.manual_seed(12)
    torch.rand(3)
    per_image = np.random.RandomState(13)
    per_image.randn(1)                                        # has_gauss = 1: the cached Gaussian must round-trip too
    eot_rng = np.random.RandomState(14)
    eot_rng.rand(7)
    A.save_checkpoint(path, dict(images=[s.state(), fresh.state()], np_global=A.rng_state_out(np.random),
                                 torch_cpu=torch.get_rng_state(), rng=A.rng_state_out(per_image),
                                 eot_rng=A.rng_state_out(eot_rng)))
    want = (_draws(np.random), torch.rand(4), _draws(per_image), _draws(eot_rng))

    np.random.seed(0)                                         # a restarted process: other stream positions
    torch.manual_seed(0)
    per_image, eot_rng = np.random.RandomState(0), np.random.RandomState(0)
    ck = torch.load(path, weights_only=True)
    A.rng_state_in(np.random, ck["np_global"])
    torch.set_rng_state(ck["torch_cpu"])
    A.rng_state_in(per_image, ck["rng"])
    A.rng_state_in(eot_rng, ck["eot_rng"])
    got = (_draws(np.random), torch.rand(4), _draws(per_image), _draws(eot_rng))
    for a, b in zip(want[0] + want[2] + want[3], got[0] + got[2] + got[3]):
        assert np.array_equal(a, b)
    assert torch.equal(want[1], got[1])

    for src, d in ((s, ck["images"][0]), (fresh, ck["images"][1])):
        r = A._ImageState(0.5, 0.0, 0, True, None)
        r.load_state(d)
        for k in ("lr", "loss_best", "not_decay", "num_failure", "coeff_group_lasso", "structured", "y", "targeted",
                  "crit_targeted", "certifiable", "active", "n_failed", "failed"):
            assert getattr(r, k) == getattr(src, k), k
        assert type(r.lr) is np.float32 and type(r.loss_best) is np.float32
    assert np.isinf(r.num_failure) and np.isinf(r.loss_best) and r.failed == []


def test_fingerprint_mismatch_names_the_field(tmp_path):
    path = str(tmp_path / "ck.pt")
    fp = _fp()
    A.save_checkpoint(path, _ckpt(fp))
    ck, digest = A.load_checkpoint(path, _fp())
    assert ck["i"] == 100 and torch.equal(ck["state"]["a"], torch.arange(5)) and digest.size == 16
    x2 = _x()
    x2[1, 2, 3, 4] += 1e-3
    for other, field in ((_fp(x=x2), "x_sha256"), (_fp(x=_x()[:1]), "x_shape"), (_fp(y=(3, 5)), "y"),
                         (_fp(lr=0.02), "lr"), (_fp(sampling_size=64), "sampling_size"), (_fp(dual=True), "dual"),
                         (_fp(eot_sampler="device"), "eot_sampler"), (_fp(image_seeds=[1, 2]), "image_seeds"),
                         (_fp(structured=0.0), "structured"), (_fp(precision="tf32"), "precision")):
        with pytest.raises(ValueError, match=r"\b%s differs" % field):
            A.load_checkpoint(path, other)


def test_wrong_format_version_is_refused(tmp_path):
    path = str(tmp_path / "ck.pt")
    A.save_checkpoint(path, _ckpt(_fp(), version=A.CHECKPOINT_VERSION + 1))
    with pytest.raises(ValueError, match="format version"):
        A.load_checkpoint(path, _fp())


def test_wrong_world_size_is_refused(tmp_path):
    path = str(tmp_path / "ck.pt")
    A.save_checkpoint(path, _ckpt(_fp(world=2)))
    with pytest.raises(ValueError, match=r"\bworld_size differs"):
        A.load_checkpoint(path, _fp(world=1))


def test_failed_write_leaves_the_previous_file(tmp_path, monkeypatch):
    path = str(tmp_path / "ck.pt")
    A.save_checkpoint(path, _ckpt(_fp()))
    before = open(path, "rb").read()

    def broken_save(obj, f, *a, **k):
        f.write(b"half a checkpoint")
        raise OSError("disk full")

    monkeypatch.setattr(torch, "save", broken_save)
    with pytest.raises(OSError, match="disk full"):
        A.save_checkpoint(path, _ckpt(_fp(), i=200))
    assert open(path, "rb").read() == before
    assert os.listdir(str(tmp_path)) == ["ck.pt"]             # the temporary file is gone too
    monkeypatch.undo()
    assert A.load_checkpoint(path, _fp())[0]["i"] == 100


def test_generate_refuses_bad_checkpoint_every():
    x = torch.zeros(1, 3, 56, 56)
    for bad in (0, -5, 2.5, True):
        with pytest.raises(ValueError, match="checkpoint_every"):
            A.DorPatch().generate(None, x, 0.12, 1000, None, 0, checkpoint="ck.pt", checkpoint_every=bad)


def test_main_flag_and_result_path(tmp_path, monkeypatch):
    from dorpatch_b200 import main as M
    from dorpatch_b200.utils import generate_saving_path
    monkeypatch.chdir(tmp_path)
    args = M.parser.parse_args([])
    assert args.checkpoint_every == 0
    on = M.parser.parse_args(["--checkpoint_every", "50"])
    assert on.checkpoint_every == 50
    assert generate_saving_path(vars(on).copy()) == generate_saving_path(vars(args).copy())
    with pytest.raises(SystemExit):
        M.parser.parse_args(["--checkpoint_every", "often"])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_worker(rank, world, port, path, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fp = _fp(world=world)
        assert A.read_checkpoint(path, fp, dist) is None        # no file yet: both ranks start fresh

        def make():
            if rank != 0:
                raise AssertionError("rank %d built a checkpoint" % rank)
            return _ckpt(fp, state=dict(a=torch.arange(5) * 3, rank=rank))

        A.write_checkpoint(path, make, dist)
        assert os.path.exists(path)                             # the barrier: in place on every rank
        ck = A.read_checkpoint(path, fp, dist)
        q.put((rank, ck["state"]["rank"], ck["state"]["a"].tolist(), ck["i"]))
        A.remove_checkpoint(path, dist)
        assert not os.path.exists(path)
    except BaseException as e:                                  # noqa: BLE001 -- reported through the queue
        q.put((rank, repr(e)))
    dist.barrier()
    dist.destroy_process_group()


def test_rank0_writes_and_every_rank_reads_world2(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    path = str(tmp_path / "adv_ckpt_0.pt")
    procs = [ctx.Process(target=_dist_worker, args=(r, 2, port, path, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, 0, [0, 3, 6, 9, 12], 100), (1, 0, [0, 3, 6, 9, 12], 100)]


def _disagree_worker(rank, world, port, path, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fp = _fp(world=world)
    mine = "%s.%d" % (path, rank)                               # each rank sees its own file: not a shared directory
    A.save_checkpoint(mine, _ckpt(fp, i=100 * (rank + 1)))
    try:
        A.read_checkpoint(mine, fp, dist)
        q.put((rank, "read"))
    except RuntimeError as e:
        q.put((rank, "same checkpoint file" in str(e)))
    dist.barrier()
    dist.destroy_process_group()


def test_ranks_reading_different_checkpoints_are_refused_world2(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_disagree_worker, args=(r, 2, port, str(tmp_path / "ck.pt"), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]
