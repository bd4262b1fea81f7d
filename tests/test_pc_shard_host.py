"""PatchCleanser evaluation sharded over the ranks of a process group, on the CPU.

The planner (attack.shard_range at the engine's chunk) covers every sample once and cuts only at chunk boundaries; the
second-round checks go round-robin in the single-process order (attack.sharded_checks); and a world-2 gloo run of
robust_predict (PatchCleanser(..., shard=True)) on a fake engine gives, on both ranks, the records of the same call without sharding
(DORPATCH_SHARD=none), while the chunks the ranks forward together are exactly the chunks the single process forwards.
A defense built without shard=True stays local under the group.  DORPATCH_AUTOTUNE reaches the Engine ResNetV2.engine()
builds."""
import collections
import contextlib
import datetime
import importlib.util
import io
import os
import pickle
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from dorpatch_b200.attack import shard_range, sharded_checks, sharded_predict

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


SIM = _load("pc_shard_sim")


def test_shard_range_covers_every_sample_once_at_chunk_boundaries():
    for n in (1, 5, 36, 63, 64, 65, 630, 2520, 22680):
        for chunk in (1, 16, 64, 128):
            for world in (1, 2, 3, 5, 8):
                sl = [shard_range(n, r, world, chunk) for r in range(world)]
                assert sl == [shard_range(n, r, world, chunk) for r in range(world)]          # same inputs, same slices
                assert np.array_equal(np.concatenate([np.arange(lo, hi) for lo, hi in sl]), np.arange(n))
                chunks = -(-n // chunk)
                for lo, hi in sl:
                    assert lo <= hi and (lo == hi or lo % chunk == 0) and (hi % chunk == 0 or hi == n)
                    assert -(-(hi - lo) // chunk) <= -(-chunks // world)                   # no rank above its share
    assert [shard_range(36, r, 2, 64) for r in range(2)] == [(0, 36), (36, 36)]             # one chunk: rank 0 alone
    assert [shard_range(630, r, 3, 128) for r in range(3)] == [(0, 256), (256, 512), (512, 630)]


def test_shard_range_unit_1_is_the_universe_scan_split():
    for n in (1, 145, 2520):
        for world in (2, 3):
            per = -(-n // world)
            assert [shard_range(n, r, world) for r in range(world)] == \
                [(min(r * per, n), min((r + 1) * per, n)) for r in range(world)]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_predict_and_checks_in_a_simulated_world(world):
    """Each rank forwards its chunk-aligned slice and gets the whole call's labels; check i runs on rank i % world only,
    and every rank gets every result in the single-process order."""
    n, chunk = 630, 64
    labels = np.random.RandomState(0).randint(0, 7, n).astype(np.int32)
    want_checks = [i % 3 == 1 for i in range(11)]

    def rank_fn(d):
        seen, ran = [], []

        def predict(lo, hi):
            seen.append((lo, hi))
            return labels[lo:hi]

        def check(i):
            ran.append(i)
            return want_checks[i]
        got = sharded_predict(predict, n, chunk, d)
        res = sharded_checks(check, len(want_checks), d)
        return got, seen, res, ran

    out = SIM.ThreadWorld(world).run(rank_fn)
    for r, (got, seen, res, ran) in enumerate(out):
        assert got.dtype == np.int32 and np.array_equal(got, labels)
        lo, hi = shard_range(n, r, world, chunk)
        assert seen == ([(lo, hi)] if hi > lo else [])
        assert res == want_checks and ran == list(range(r, len(want_checks), world))
    assert sharded_checks(lambda i: want_checks[i], len(want_checks)) == want_checks


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _BoolWindow:
    def __init__(self, single, double):
        self.mask_set, self.double_mask_set = single, double


def _cases():
    """(name, window, rectangle window the fake decodes with, chunk)."""
    from dorpatch_b200.defenses.PatchCleanser import MaskWindow
    with contextlib.redirect_stdout(io.StringIO()):
        one, two = MaskWindow(56, 0.12, 1), MaskWindow(56, 0.12, 2)
    return [("one_patch_c64", one, one, 64), ("one_patch_c16", one, one, 16), ("two_patch_c128", two, two, 128),
            ("two_patch_c64", two, two, 64), ("bank_one_patch_c16", _BoolWindow(one.mask_set, one.double_mask_set), one, 16)]


def _evaluate(pc, fake, img, certify, shard):
    os.environ["DORPATCH_SHARD"] = "eot" if shard else "none"
    fake.chunks.clear()
    rec = pc.robust_predict(img, certify)
    return rec, list(fake.chunks)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    # a rank left alone in a collective fails after a minute instead of waiting for the default half hour
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))
    from dorpatch_b200.defenses.PatchCleanser import PatchCleanser
    from dorpatch_b200.resnetv2 import ResNetV2
    net = ResNetV2()
    img = torch.rand(3, 56, 56, generator=torch.Generator().manual_seed(0))
    failures, covered = [], set()
    try:
        for name, window, mw, chunk in _cases():
            n1, n2 = len(mw.mask_rects), len(mw.double_mask_rects)
            for sname, first, second, cert in SIM.scenarios(n1, n2):
                fake = SIM.FakeEngine(chunk, mw, first, second, cert)
                pc = PatchCleanser(window, net, shard=True)
                pc._engine = lambda im: fake
                expected, confirmed = SIM.expected_prediction(first, second)
                for certify in (True, False):
                    tag = "%s/%s/certify=%s" % (name, sname, certify)
                    want, want_chunks = _evaluate(pc, fake, img, certify, False)
                    got, my_chunks = _evaluate(pc, fake, img, certify, True)
                    everyone = [None] * world
                    dist.all_gather_object(everyone, my_chunks)
                    union = collections.Counter(c for chunks in everyone for c in chunks)
                    if not SIM.records_equal(got, want) or pickle.dumps(got) != pickle.dumps(want):
                        failures.append(tag + ": records differ")
                    if union != collections.Counter(want_chunks):
                        failures.append(tag + ": the ranks forwarded other chunks than one process")
                    if want.prediction != expected or got.prediction != expected:
                        failures.append(tag + ": prediction %r / %r, the reference's rule gives %r"
                                        % (want.prediction, got.prediction, expected))
                    if sname == "round2" and len(confirmed) < 2:
                        failures.append(tag + ": scenario does not confirm two labels (%s)" % confirmed)
                    covered.add((name.split("_c")[0], sname, certify, want.preds_2 is not None))
        # a defense built without shard=True stays local under the group: rank 0 alone evaluates, with the calls and
        # the record of one process, while rank 1 enters no collective until the barrier below
        name, window, mw, chunk = _cases()[2]
        sname, first, second, cert = SIM.scenarios(len(mw.mask_rects), len(mw.double_mask_rects))[2]
        fake = SIM.FakeEngine(chunk, mw, first, second, cert)
        pc = PatchCleanser(window, net)
        pc._engine = lambda im: fake
        if pc._group() is not None:
            failures.append("a defense without shard=True joins the process group")
        if rank == 0:
            want, want_chunks = _evaluate(pc, fake, img, True, False)
            got, chunks = _evaluate(pc, fake, img, True, True)
            if not SIM.records_equal(got, want) or chunks != want_chunks:
                failures.append("a defense without shard=True differs from one process on rank 0 alone")
    except BaseException as ex:
        failures.append("rank %d raised %r" % (rank, ex))
    q.put((rank, failures, sorted(covered)))
    dist.barrier()
    dist.destroy_process_group()


def test_robust_predict_world2_gloo_equals_one_process():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert [r for r, _, _ in res] == [0, 1]
    for r, failures, _ in res:
        assert failures == [], (r, failures)
    covered = res[0][2]
    assert {w for w, _, _, _ in covered} == {"one_patch", "two_patch", "bank_one_patch"}
    assert ("two_patch", "round2", False, False) in covered and ("two_patch", "round2", True, True) in covered


def test_autotune_env_reaches_the_engine(monkeypatch):
    import dorpatch_b200.engine as E
    from dorpatch_b200 import runtime
    from dorpatch_b200.resnetv2 import ResNetV2
    made = []

    class _Engine:
        def __init__(self, **kw):
            made.append(kw)
            self.max_images, self.handle = kw["max_images"], True

        def load_state_dict(self, sd):
            pass

        def close(self):
            pass

    monkeypatch.setattr(E, "Engine", _Engine)
    monkeypatch.setattr(runtime, "register", lambda e: None)
    net = ResNetV2()
    monkeypatch.delenv("DORPATCH_AUTOTUNE", raising=False)
    net.engine(56)
    monkeypatch.setenv("DORPATCH_AUTOTUNE", "0")
    net.engine(112)
    monkeypatch.setenv("DORPATCH_AUTOTUNE", "1")
    net.engine(168)
    assert [kw["autotune"] for kw in made] == [True, False, True]
