"""The on-device EOT draw (dp_eot_draw, DorPatch.generate(eot_sampler="device")) on the GPU: the kernel against its numpy
restatement (tests/test_device_sampler_host.py) bit for bit, the sampling invariants, the rectangles against
masks.gather, reproducibility across engines, batch sizes, rank slices and graph replay, uniformity, and a generate()
run whose only difference from the host path is where the draws come from."""
import importlib.util
import os

import numpy as np
import pytest
import torch
from scipy import stats

from dorpatch_b200 import masks as PM

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("device_sampler_host", os.path.join(HERE, "test_device_sampler_host.py"))
REF = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(REF)

# (dropout, n_patch) -> universe size at any image size: 144, 2520, 2520, 90720
UNIVERSES = [(1, 1), (2, 1), (1, 2), (2, 2)]


def _engine(params, precision="fp32", chunk=8, max_images=4):
    """An engine of this module's own.  Every engine the module creates is closed before pytest moves on, so the suite's
    later modules find the device memory free (each engine holds two 512 MB library workspaces)."""
    from dorpatch_b200.engine import Engine
    e = Engine(img=112, precision=precision, chunk=chunk, max_images=max_images, autotune=False)
    e.load_state_dict(params)
    return e


@pytest.fixture(scope="module")
def eng(oracle_params):
    e = _engine(oracle_params)
    yield e
    e.close()


def _setup(e, table, sets):
    e.failed_reset(len(table))
    e.eot_universe(table)
    for b, f in enumerate(sets):
        e.failed_write(b, f)


def _sets(rng, n, S):
    """Four failed sets: empty, smaller than S/2, sparse, dense."""
    return [[], sorted(rng.choice(n, S // 2 - 3, replace=False).tolist()),
            sorted(rng.choice(n, min(n, 3 * S), replace=False).tolist()),
            sorted(rng.choice(n, n // 2, replace=False).tolist())]


@pytest.mark.parametrize("dropout,n_patch", UNIVERSES)
def test_draw_invariants_and_reference(eng, dropout, n_patch):
    table = PM.universe(112, dropout, n_patch)
    n = len(table)
    duals = (False, True) if table.shape[1] <= 2 else (False,)
    rng = np.random.RandomState(dropout * 10 + n_patch)
    for S in (32, min(128, n)):
        sets = _sets(rng, n, S)
        _setup(eng, table, sets)
        for dual in duals:
            for stage, it in ((0, 999), (1, 1000), (0, 1234), (1, 4999)):
                seeds = rng.randint(0, 2 ** 62, size=4)
                idx, idx2, nff = eng.eot_draw(seeds, stage, it, [1, 1, 1, 1], S, dual, host=True)
                for b in range(4):
                    want_ff = 0 if it < 1000 else min(len(sets[b]), S // 2)
                    assert nff[b] == want_ff
                    assert set(eng.failed_read(b)) == set(sets[b])
                    for row in ([idx[b]] + ([idx2[b]] if dual else [])):
                        ff, uni = row[:want_ff], row[want_ff:]
                        assert len(set(ff.tolist())) == len(ff) and len(set(uni.tolist())) == len(uni)
                        assert set(ff.tolist()) <= set(sets[b])
                        assert uni.min() >= 0 and uni.max() < n
                    r_idx, r_idx2, r_ff = REF.reference_draw(seeds[b], stage, it, sets[b], n, S, dual)
                    assert r_ff == nff[b]
                    assert np.array_equal(idx[b], r_idx), (b, stage, it)
                    if dual:
                        assert np.array_equal(idx2[b], r_idx2)


def test_inactive_images_untouched(eng):
    table = PM.universe(112, 2)
    rng = np.random.RandomState(5)
    _setup(eng, table, _sets(rng, len(table), 32))
    before = eng.eot_draw([1, 2, 3, 4], 1, 1200, [1, 1, 1, 1], 32, True, host=True)
    after = eng.eot_draw([9, 9, 9, 9], 1, 1300, [0, 1, 0, 1], 32, True, host=True)
    for b in (0, 2):
        assert np.array_equal(before[0][b], after[0][b]) and np.array_equal(before[1][b], after[1][b])
        assert before[2][b] == after[2][b]
    for b in (1, 3):
        assert not np.array_equal(before[0][b], after[0][b])


@pytest.mark.parametrize("dropout,n_patch,dual", [(2, 1, False), (2, 1, True), (1, 2, True), (2, 2, False)])
def test_rectangles_equal_gather(eng, dropout, n_patch, dual):
    table = PM.universe(112, dropout, n_patch)
    rng = np.random.RandomState(11)
    _setup(eng, table, _sets(rng, len(table), 48))
    for world, rank in ((1, 0), (2, 1), (3, 2)):
        idx, idx2, _ = eng.eot_draw([5, 6, 7, 8], 1, 1100, [1, 1, 1, 1], 48, dual, rank, world, host=True)
        s_loc = 48 // world
        sl = slice(rank * s_loc, (rank + 1) * s_loc)
        want = PM.gather(table, idx[:, sl], idx2[:, sl] if dual else None).reshape(-1, 4, 4)
        assert np.array_equal(eng.eot_draw_rects(4 * s_loc), want)


def test_reproducible_across_engines_batch_and_ranks(eng, oracle_params):
    table = PM.universe(112, 2)
    rng = np.random.RandomState(3)
    sets = _sets(rng, len(table), 48)
    seeds = [11, 2 ** 40 + 5, 77, 123456789]
    other = _engine(oracle_params, precision="bf16", chunk=16)
    try:
        draws = []
        for e in (eng, other):
            _setup(e, table, sets)
            draws.append(e.eot_draw(seeds, 1, 1500, [1, 1, 1, 1], 48, True, host=True))
        for a, b in zip(*draws):
            assert np.array_equal(a, b)
        idx, idx2, nff = draws[0]
        for b in range(4):                                 # row b of the B = 4 draw = a B = 1 draw seeded s_b
            _setup(other, table, [sets[b]])
            one = other.eot_draw([seeds[b]], 1, 1500, [1], 48, True, host=True)
            assert np.array_equal(one[0][0], idx[b]) and np.array_equal(one[1][0], idx2[b]) and one[2][0] == nff[b]
    finally:
        other.close()
    _setup(eng, table, sets)
    eng.eot_draw(seeds, 1, 1500, [1, 1, 1, 1], 48, True)
    whole = eng.eot_draw_rects(4 * 48).reshape(4, 48, 4, 4)
    for world in (2, 3, 8):                                # the rank slices concatenate to the world-1 rectangles
        parts = []
        for rank in range(world):
            got = eng.eot_draw(seeds, 1, 1500, [1, 1, 1, 1], 48, True, rank, world, host=True)
            assert np.array_equal(got[0], idx) and np.array_equal(got[1], idx2)
            parts.append(eng.eot_draw_rects(4 * 48 // world).reshape(4, 48 // world, 4, 4))
        assert np.array_equal(np.concatenate(parts, 1), whole)


def _steps(e, x, mask, pattern, y, table, B, S, n_steps, seeds):
    """n_steps device-sampler steps (draw, gradient, failed-set update, sign step) at i >= 1000; per step the drawn
    indices, the losses and the set sizes."""
    G = torch.zeros_like(x)
    out = []
    for i in range(1000, 1000 + n_steps):
        idx, _, nff = e.eot_draw(seeds, 1, i, [1] * B, S, host=True)
        r = e.attack_grad(x, mask, pattern, None, y, [True] * B, 0.1, 4.0, 1, G, S_total=S, S=S)
        cnt = e.failed_update_drawn(B, S, [1] * B)
        e.attack_update(x, mask, pattern, G, np.full(B, 0.01, np.float32), [1e-3] * B, [1e-5] * B, 1e-3, 1)
        out.append((idx.copy(), nff.copy(), r["loss_adv"].copy(), cnt.copy()))
    return out


def _step_inputs(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 3, 112, 112, generator=g).cuda()
    pattern = torch.rand(B, 3, 112, 112, generator=g).cuda()
    mask = (torch.rand(B, 1, 112, 112, generator=g) > 0.7).float().cuda()
    return x, mask, pattern


def test_graph_replay_matches_plain_launches(oracle_params, monkeypatch):
    """B = 1 x S = 128: device-sampler steps replay the step's CUDA graph, and give the bits of an engine that
    launches everything plainly (DORPATCH_GRAPH=0)."""
    table = PM.universe(112, 2)
    e = _engine(oracle_params, chunk=32, max_images=1)
    monkeypatch.setenv("DORPATCH_GRAPH", "0")
    plain = _engine(oracle_params, chunk=32, max_images=1)
    monkeypatch.delenv("DORPATCH_GRAPH")
    runs = []
    try:
        for k, en in enumerate((e, plain)):
            _setup(en, table, [list(range(0, 2520, 9))])
            x, mask, pattern = _step_inputs(1)
            r0 = en.graph_replays
            runs.append(_steps(en, x, mask, pattern, [3], table, 1, 128, 5, [99]))
            if k == 0:
                assert en.graph_replays - r0 >= 4, (en.graph_replays - r0, en.graph_status)
            else:
                assert en.graph_replays == r0
    finally:
        e.close()
        plain.close()
    for a, b in zip(*runs):
        for u, v in zip(a, b):
            assert np.array_equal(u, v)
    assert any(s[1][0] > 0 for s in runs[0])             # the failed part was drawn


def test_uniformity_chi_squared(eng):
    """Fixed seeds, so deterministic.  Threshold: the chi-squared quantile at 1 - 1e-6 for the bins' degrees of
    freedom (a correct sampler fails one run in a million seeds; this seed is fixed)."""
    q = 1 - 1e-6
    table = PM.universe(112, 2)
    n, S = len(table), 128
    members = list(range(5, 2520, 63))                    # sparse failed set: 40 of 2520
    _setup(eng, table, [[], members, [], []])
    count_uni = np.zeros(n)
    count_first = np.zeros(20)                            # the first position alone, 20 bins of 126 indices
    count_ff = np.zeros(len(members))
    pos = {m: k for k, m in enumerate(members)}
    draws = 0
    for step in range(500):
        idx, _, nff = eng.eot_draw([1000 + step, 2000 + step, 3000 + step, 4000 + step], 0, step, [1, 1, 1, 1], S,
                                   host=True)
        for b in (0, 2, 3):                               # universe part: i < 1000
            np.add.at(count_uni, idx[b], 1)
            count_first[idx[b][0] // 126] += 1
        draws += 3
        idx, _, nff = eng.eot_draw([5000 + step, 1, 2, 3], 1, 1000 + step, [0, 1, 0, 0], 32, host=True)
        assert nff[1] == 16                               # min(|F| = 40, S/2): 16 of the 40 members per draw
        for m in idx[1][:nff[1]]:
            count_ff[pos[int(m)]] += 1
    assert draws >= 1500 and count_ff.sum() == 500 * 16
    exp = draws * S / n
    chi = ((count_uni - exp) ** 2 / exp).sum()
    assert chi < stats.chi2.ppf(q, n - 1), chi
    exp = draws / 20
    chi = ((count_first - exp) ** 2 / exp).sum()
    assert chi < stats.chi2.ppf(q, 19), chi
    exp = count_ff.sum() / len(members)
    chi = ((count_ff - exp) ** 2 / exp).sum()
    assert chi < stats.chi2.ppf(q, len(members) - 1), chi


def _expect_refusal(fn, what):
    with pytest.raises(RuntimeError, match=what):
        fn()


@pytest.fixture
def fresh(oracle_params):
    from dorpatch_b200.engine import Engine
    e = Engine(img=112, precision="fp32", chunk=8, max_images=2, autotune=False)
    e.load_state_dict(oracle_params)
    yield e
    e.close()


def test_refuses_draw_before_upload(fresh):
    _expect_refusal(lambda: fresh.eot_draw([1], 0, 0, [1], 32), "no universe")


def test_refuses_S_above_n_mask(fresh):
    table = PM.universe(112, 1)                           # 144 masks
    _setup(fresh, table, [])
    fresh.eot_draw([1], 0, 0, [1], 144)                   # S = n_mask is exact
    _expect_refusal(lambda: fresh.eot_draw([1], 0, 0, [1], 145), "outside")


def test_refuses_universe_larger_than_sets(fresh):
    fresh.failed_reset(144)
    fresh.eot_universe(PM.universe(112, 2))               # 2520 masks
    _expect_refusal(lambda: fresh.eot_draw([1], 0, 0, [1], 32), "exceed the failed-set bitmaps")


def test_refuses_stale_draw(fresh):
    table = PM.universe(112, 2)
    _setup(fresh, table, [[1, 2, 3]])
    x, mask, pattern = _step_inputs(1)
    G = torch.zeros_like(x)
    grad = lambda: fresh.attack_grad(x, mask, pattern, None, [3], [True], 0.1, 4.0, 1, G, S_total=16, S=16)  # noqa: E731
    fresh.eot_draw([4], 1, 1000, [1], 16)
    grad()
    fresh.failed_update_drawn(1, 16, [1])
    _expect_refusal(grad, "no fresh")                     # the draw served its step
    _expect_refusal(lambda: fresh.failed_update_drawn(1, 16, [1]), "no fresh")
    fresh.eot_draw([4], 1, 1001, [1], 16)
    fresh.eot_universe(table)                             # a new universe invalidates the draw
    _expect_refusal(grad, "no fresh")


# ---- generate(): the two paths differ only in where the draws come from -------------------------------------------
@pytest.fixture(scope="module")
def native_model(oracle_params):
    """fp32, chunk 16.  At teardown the environment is restored and every engine created meanwhile (the model's, and
    any weight-free helper engine) is closed."""
    from dorpatch_b200 import runtime
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    saved = {k: os.environ.get(k) for k in ("DORPATCH_PRECISION", "DORPATCH_CHUNK")}
    os.environ["DORPATCH_PRECISION"], os.environ["DORPATCH_CHUNK"] = "fp32", "16"
    before = list(runtime._ENGINES)
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    yield torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()
    for e in [e for e in runtime._ENGINES if all(e is not o for o in before)] + [ent[0] for ent in net._engines.values()]:
        e.close()
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _record(monkeypatch, log):
    from dorpatch_b200.engine import Engine
    draw, grad, upd, upd_d = Engine.eot_draw, Engine.attack_grad, Engine.failed_update, Engine.failed_update_drawn

    def eot_draw(self, seeds, stage, i, active, S, dual=False, rank=0, world=1, host=False):
        got = draw(self, seeds, stage, i, active, S, dual, rank, world, host=True)
        log["draws"].append((np.asarray(active, bool), got))
        return got if host else None

    def attack_grad(self, *a, **k):
        r = grad(self, *a, **k)
        log["loss"].append(r["loss_adv"].copy())
        return r

    def failed_update(self, *a, **k):
        c = upd(self, *a, **k)
        log["counts"].append(c.copy())
        return c

    def failed_update_drawn(self, *a, **k):
        c = upd_d(self, *a, **k)
        log["counts"].append(c.copy())
        return c

    monkeypatch.setattr(Engine, "eot_draw", eot_draw)
    monkeypatch.setattr(Engine, "attack_grad", attack_grad)
    monkeypatch.setattr(Engine, "failed_update", failed_update)
    monkeypatch.setattr(Engine, "failed_update_drawn", failed_update_drawn)


@pytest.mark.parametrize("dual,pc_n_patch,dropout", [(False, 1, 2), (True, 1, 2), (False, 2, 1)])
def test_generate_device_equals_host_with_the_same_draws(native_model, monkeypatch, dual, pc_n_patch, dropout):
    from dorpatch_b200 import attack as A
    g = torch.Generator().manual_seed(21)
    x = torch.rand(2, 3, 112, 112, generator=g).cuda()
    kw = dict(max_iterations=8, sampling_size=32, dual=dual, pc_n_patch=pc_n_patch, dropout=dropout)

    def run(sampler):
        torch.manual_seed(5)
        np.random.seed(5)
        log = dict(draws=[], loss=[], counts=[])
        with monkeypatch.context() as mp:
            _record(mp, log)
            if sampler == "host":                         # _ImageState.sample returns the device run's draws, in order
                queue = {b: [] for b in range(2)}
                for active, (idx, idx2, nff) in dev_log["draws"]:
                    for b in np.nonzero(active)[0]:
                        queue[b].append((idx[b].astype(np.int64), int(nff[b])))
                        if dual:
                            queue[b].append((idx2[b].astype(np.int64), int(nff[b])))
                mp.setattr(A._ImageState, "sample", lambda self, i, n_mask, S: queue[self.dev[1]].pop(0))
            m, p = A.DorPatch().generate(native_model, x, 0.12, 1000, None, 0, eot_sampler=sampler, **kw)
            if sampler == "host":
                assert all(len(q) == 0 for q in queue.values())
        return m, p, log

    dev_m, dev_p, dev_log = run("device")
    host_m, host_p, host_log = run("host")
    assert len(dev_log["draws"]) == 16
    assert torch.equal(dev_m, host_m) and torch.equal(dev_p, host_p)
    assert len(dev_log["loss"]) == len(host_log["loss"])
    for a, b in zip(dev_log["loss"], host_log["loss"]):
        assert np.array_equal(a, b)
    for a, b in zip(dev_log["counts"], host_log["counts"]):
        assert np.array_equal(a, b)
