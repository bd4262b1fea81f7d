"""basic_unit other than 7 on the GPU: the density / group-lasso regulariser and the stage-0 mask gradient against the
oracle at every unit, patch_selection, generate against the oracle, the unit as part of the CUDA-graph signature, and the
main.py driver with --basic_unit."""
import contextlib
import io
import os
import random

import numpy as np
import pytest
import torch

from oracle import attack as OA, resnetv2 as OR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UNITS = [(56, u) for u in (1, 2, 4, 7, 8, 14, 28, 56)] + [(224, u) for u in (1, 2, 4, 8, 14, 16, 28, 32)]


def _seed(s=1234):
    random.seed(s)
    torch.manual_seed(s)
    np.random.seed(s)


def _masks(H, u, seed):
    """B = 3 masks in [0, 1] with exact zeros: image 0 an all-zero group in its corner, image 1 about 5 % zero pixels
    (each an all-zero group at u = 1), image 2 an all-zero band of u rows, plus a zero density window."""
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(3, 1, H, H, generator=g)
    m[0, 0, :u, :u] = 0
    m[1][torch.rand(1, H, H, generator=g) < 0.05] = 0
    m[2, 0, H - u:, :] = 0
    m[2, 0, :H // 8, :H // 8] = 0
    return m


@pytest.fixture(scope="module")
def native_model(oracle_params):
    from dorpatch_b200.resnetv2 import ResNetV2
    from dorpatch_b200.utils import NormModel, get_normalize
    os.environ["DORPATCH_PRECISION"] = "fp32"
    os.environ["DORPATCH_CHUNK"] = "16"
    net = ResNetV2(seed=0)
    net.load_state_dict(oracle_params)
    return torch.nn.DataParallel(NormModel(net, get_normalize("imagenet", "resnetv2"))).cuda().eval()


@pytest.mark.parametrize("H,u", UNITS)
def test_regularisers_and_stage0_mask_gradient_match_oracle(engine_factory, H, u):
    """loss_density, group_lasso and grad_mask_out of dp_attack_update at basic_unit u, fp32, B = 3, against the oracle
    in float64.  pattern == x makes the classifier's share of the mask gradient exactly 0, so grad_mask_out is
    density * d var / d m + coeff * u * m / sqrt(group sum of squares).  Values to fp32 rounding; the sign of every
    pixel's gradient equal, zeros included (NaN for an all-zero group, quirk Q5, has sign 0 and leaves the pixel)."""
    B = 3
    e = engine_factory(img=H, precision="fp32", chunk=4, max_images=B)
    x = torch.rand(B, 3, H, H, generator=torch.Generator().manual_seed(u))
    m = _masks(H, u, 100 + u)
    rects = np.zeros((B, 1, 4, 4), np.int16)
    for density, coeff in ((1e-3, 1e-5), (0.0, 3e-5)):
        xd, md, pd = x.to(DEV), m.to(DEV).clone(), x.to(DEV).clone()
        G = torch.zeros(B, 3, H, H, device=DEV)
        r = e.attack_grad(xd, md, pd, rects, np.array([1, 2, 3]), [True, False, True], 0.1, 4.0, 0, G, basic_unit=u)
        gm = torch.zeros_like(md)
        lr = np.full(B, 0.01, np.float32)
        e.attack_update(xd, md, pd, G, lr, [1e-3] * B, [coeff] * B, density, 0, grad_mask_out=gm)
        torch.cuda.synchronize()

        m64 = m.double().requires_grad_(True)
        dens, gl = OA.density_loss(m64, H // 8), OA.group_lasso(m64, u)
        (density * dens + coeff * gl).sum().backward()
        ref = m64.grad.float()
        assert np.allclose(r["loss_density"], dens.detach().numpy(), rtol=2e-5, atol=1e-6), (r["loss_density"], dens)
        assert np.allclose(r["group_lasso"], gl.detach().numpy(), rtol=2e-5), (r["group_lasso"], gl)
        got = gm.cpu()
        nan_ref = torch.isnan(ref)
        assert torch.equal(torch.isnan(got), nan_ref)
        assert int(nan_ref.sum()) > 0
        fin = ~nan_ref
        scale = ref[fin].abs().max().item()
        err = (got[fin] - ref[fin]).abs()
        assert (err <= 1e-5 * scale + 1e-4 * ref[fin].abs()).all(), err.max().item()
        sref, sgot = torch.nan_to_num(ref).sign(), torch.nan_to_num(got).sign()
        if density == 0:       # one term, no cancellation: every sign is pinned
            decided = torch.ones_like(nan_ref)
        else:                  # a pixel where the two terms cancel to within fp32 rounding is a tie either way
            decided = (ref.abs() > 1e-5 * scale) | (ref == 0) | nan_ref
            assert int((~decided).sum()) <= 0.01 * ref.numel()
        assert torch.equal(sgot[decided], sref[decided]), int((sgot != sref)[decided].sum())
        # the sign step, NaN pixels frozen
        assert torch.equal(md.cpu(), (m - 0.01 * sgot).clamp(0, 1))


@pytest.mark.parametrize("H,u", UNITS)
def test_patch_selection_matches_oracle(H, u):
    """DorPatch.patch_selection(mask, budget, u) (device window sums, host top-k) == the oracle's."""
    from dorpatch_b200.attack import DorPatch
    m = _masks(H, u, 200 + u)
    for budget in (0.06, 0.12):
        got = DorPatch().patch_selection(m.to(DEV), budget, u)
        assert torch.equal(got.cpu(), OA.patch_selection(m, budget, u)), budget


def _generate(model, x, save_dir, **kw):
    from dorpatch_b200.attack import DorPatch
    _seed()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        m, p = DorPatch().generate(model, x.cuda(), save_dir=save_dir, batch_id=0, **kw)
    log = [l for l in buf.getvalue().splitlines() if not l.startswith("mask size")]
    return m.cpu(), p.cpu(), log, np.random.get_state()[1][:4].copy()


@pytest.mark.parametrize("u,budget", [(4, 0.12), (14, 0.30)])
def test_generate_basic_unit_matches_oracle(native_model, oracle_params, tmp_path, u, budget):
    """generate(basic_unit=u) at fp32, 112 px, targeted, 2 stages x 3 iterations, S = 8, against the oracle on the same
    seeds: identical numpy RNG consumption and log structure, patch mask IoU >= 0.90, at most 5 % of the pattern's pixels
    off by more than lr/4 (sign(grad) steps of last-bit gradient differences, as in test_gpu_generate._compare).  At
    u = 14 the budget selects 19 of 64 groups, so that one group on either side of a near-tie keeps IoU >= 0.90."""
    H, LR = 112, 0.01
    x = torch.rand(1, 3, H, H, generator=torch.Generator().manual_seed(17))
    kw = dict(patch_budget=budget, n_classes=1000, targeted=True, max_iterations=3, sampling_size=8, dropout=1, lr=LR,
              basic_unit=u)
    tgt = torch.tensor([321])
    m_gpu, p_gpu, log_gpu, rng_gpu = _generate(native_model, x, str(tmp_path / "c" / "sub"), y=tgt.cuda(), **kw)
    net = OR.OracleNet(oracle_params, weights_require_grad=False).eval()
    _seed()
    log_or = []
    m_or, p_or = OA.generate(net, x, y=tgt, log=log_or.append, **kw)
    rng_or = np.random.get_state()[1][:4].copy()
    assert np.array_equal(rng_gpu, rng_or)
    assert len(log_gpu) == len(log_or)
    for a, b in zip(log_gpu, log_or):
        print("GPU:", a)
        print("ORA:", b)
        assert a.split(",")[0] == b.split(",")[0]
    # the selected patch is made of whole u x u cells
    cells = m_gpu.reshape(H // u, u, H // u, u)
    assert torch.equal(cells, cells[:, :1, :, :1].expand_as(cells))
    inter = ((m_gpu > 0.5) & (m_or > 0.5)).sum().item()
    union = ((m_gpu > 0.5) | (m_or > 0.5)).sum().item()
    iou = inter / max(union, 1)
    frac = ((p_gpu - p_or).abs() > 0.25 * LR).float().mean().item()
    print("mask IoU", iou, "pattern pixels off by > lr/4", frac)
    assert iou >= 0.90 and frac <= 0.05, (iou, frac)


def test_basic_unit_is_part_of_the_graph_signature(oracle_params, monkeypatch):
    """With CUDA graphs on, stage 0 at u = 7 is captured and replayed; a following call at u = 14 with the same tensors
    must not replay the u = 7 graph: it equals a graphs-off engine's u = 14 call bit for bit (patch gradient, losses,
    regularisers and the mask gradient of the update that follows)."""
    from dorpatch_b200.engine import Engine
    H, B, S = 112, 2, 4
    g = torch.Generator().manual_seed(5)
    x, m, p = torch.rand(B, 3, H, H, generator=g), _masks(H, 14, 6)[:B], torch.rand(B, 3, H, H, generator=g)
    rects = np.zeros((B, S, 4, 4), np.int16)
    rects[:, :, 0] = [10, 40, 20, 50]
    y = np.array([3, 9])

    def call(e, xd, md, pd, G, u):
        r = e.attack_grad(xd, md, pd, rects, y, [True, False], 0.1, 4.0, 0, G, basic_unit=u)
        gm = torch.zeros(B, 1, H, H, device=DEV)
        e.attack_update(xd, md, pd, G, np.zeros(B, np.float32), [1e-3] * B, [1e-5] * B, 1e-3, 0, grad_mask_out=gm)
        torch.cuda.synchronize()
        return [G.cpu(), gm.cpu()] + [torch.from_numpy(r[k].copy()) for k in ("loss_adv", "preds", "loss_struc",
                                                                               "loss_density", "group_lasso", "l2")]

    out = {}
    for graph in ("1", "0"):
        monkeypatch.setenv("DORPATCH_GRAPH", graph)
        e = Engine(img=H, precision="fp32", chunk=4, max_images=B, autotune=False)
        e.load_state_dict(oracle_params)
        xd, md, pd = x.to(DEV), m.to(DEV), p.to(DEV)
        G = torch.zeros(B, 3, H, H, device=DEV)                   # the graph signature includes the tensors
        if graph == "1":
            for _ in range(3):
                call(e, xd, md, pd, G, 7)
            assert e.graph_replays == 2, e.graph_status           # captured on call 2, replayed on call 3
            before = e.graph_replays
        out[graph] = call(e, xd, md, pd, G, 14)
        if graph == "1":
            assert e.graph_replays == before                      # a new signature runs eagerly first
        e.close()
    for a, b in zip(out["1"], out["0"]):
        assert a.numpy().tobytes() == b.numpy().tobytes()       # bitwise: the mask gradient holds NaN groups


def test_main_driver_basic_unit(tmp_path, monkeypatch):
    """main.py --basic_unit 14 end to end (bf16, 56 px): patches and records under the `__basic_unit=14` directory, the
    stage-0 cache in its parent; a later default run in the same root uses its own directory and neither reads nor
    rewrites the unit-14 artefacts."""
    from dorpatch_b200 import main as M
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("DORPATCH_PRECISION", "bf16")
    base = ["--synthetic", "2", "--random_init", "--img_size", "56", "--max_iterations", "150", "--sampling_size", "16"]

    def run(extra):
        with contextlib.redirect_stdout(io.StringIO()):
            return M.cli(base + extra)

    u14 = run(["--basic_unit", "14"])
    rd = u14["result_dir"]
    assert rd.split(os.sep)[1].endswith("_basic_unit=14") and rd.endswith("num_patch=-1_patch_budget=0.12")
    assert u14["line"].startswith("clean accuracy: ")
    stored = [os.path.join(rd, f % i) for i in range(2) for f in ("adv_mask_%d.pt", "adv_pattern_%d.pt", "adv_PC_%d.pt")]
    stored += [os.path.join(os.path.dirname(rd), f % i) for i in range(2) for f in ("adv_mask_%d.pt", "adv_pattern_%d.pt")]
    for f in stored:
        assert os.path.exists(f), f
    for i in range(2):                                            # the patch is made of whole 14 x 14 cells
        mk = torch.load(os.path.join(rd, "adv_mask_%d.pt" % i)).cpu()
        cells = mk.reshape(mk.shape[0], 4, 14, 4, 14)
        assert torch.equal(cells, cells[:, :, :1, :, :1].expand_as(cells))
    mtimes = {f: os.stat(f).st_mtime_ns for f in stored}

    loaded = []
    real_load = torch.load
    monkeypatch.setattr(torch, "load", lambda f, *a, **k: (loaded.append(os.path.abspath(str(f))), real_load(f, *a, **k))[1])
    default = run([])
    assert "basic_unit" not in default["result_dir"]
    assert os.path.dirname(default["result_dir"]) != os.path.dirname(rd)
    for i in range(2):
        assert os.path.exists(os.path.join(default["result_dir"], "adv_mask_%d.pt" % i))
    suffixed = os.path.abspath(os.path.dirname(rd))
    assert not [f for f in loaded if f.startswith(suffixed + os.sep)], loaded
    assert {f: os.stat(f).st_mtime_ns for f in stored} == mtimes
    assert sorted(os.listdir(rd)) == sorted(os.path.basename(f) for f in stored[:6])
