"""Oracle restatement of the DorPatch optimisation loop (torch-CPU, fp32).

Follows reference attack.py (CW_loss :10-23, local_variance :33-39,
min_var_weighted_variance :41-45, DorPatch.generate :51-361, patch_selection
:363-382, collect_failure :384-406) and reference utils.py:105-110 (clip).

Differences from the reference, all deliberate and documented in DESIGN.md:
  * B > 1 is defined as B independent single-image problems (the reference is
    batch-size-1 only, SURVEY quirk Q2): every piece of scalar state
    (lr, loss_best, not_decay, num_failure, failed_idxs, coeff_group_lasso,
    structured, target label, numpy RNG stream) is kept per image.  For B == 1
    the control flow, RNG consumption and arithmetic equal the reference's.
  * the two ``set_target(preds_adv)`` call sites with the wrong arity
    (attack.py:155,359 -- a TypeError in the reference, quirk Q1) call
    ``set_target(preds_adv, y)`` instead of crashing.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import os

import numpy as np
import torch

from . import masks as omasks

PATIENCE = 200                     # attack.py:65
SCALE_UP = 1.2                     # attack.py:88
SCALE_DOWN = np.sqrt(SCALE_UP ** 3)  # attack.py:89


# ----------------------------------------------------------------------------
# elementary pieces
# ----------------------------------------------------------------------------
def clip_paste(mask, pattern, x, eps):
    """utils.py:105-110: delta = m*(p-x) scaled so ||delta||_2 <= eps (norm detached)."""
    delta = mask * (pattern - x)
    l2 = torch.norm(delta, p=2, dim=(1, 2, 3)).detach()
    scale = (eps / l2).clamp(max=1.0).view(-1, 1, 1, 1)
    return delta * scale


def occlude(img, keep):
    """attack.py:206 / PatchCleanser.py:99-100: img*M + 0.5*~M (M bool, True=keep)."""
    return img * keep + 0.5 * (~keep)


def cw_loss(logits, y, num_classes, targeted, confidence):
    """attack.py:16-23."""
    onehot = torch.nn.functional.one_hot(y, num_classes)
    real = (logits * onehot).sum(1)
    other = ((1.0 - onehot) * logits - onehot * 1e4).max(1)[0]
    if targeted:                      # same association order as the reference: (conf + other) - real
        return torch.clamp(confidence + other - real, min=0.0)
    return torch.clamp(confidence + real - other, min=0.0)


def local_variance(x):
    """attack.py:33-39.  The reference subtracts in place on a *detached clone*,
    so (i) gradients flow only through the subtracted neighbour and (ii) the last
    column / row keep the raw (detached, un-abs'd) pixel value (quirk Q4)."""
    xd = x.detach()
    lr = torch.cat([(xd[..., :, :-1] - x[..., :, 1:]).abs(), xd[..., :, -1:]], dim=-1)
    ud = torch.cat([(xd[..., :-1, :] - x[..., 1:, :]).abs(), xd[..., -1:, :]], dim=-2)
    return lr + ud, lr, ud


def min_var_weighted_variance(x):
    """attack.py:41-45."""
    lv, lr, ud = local_variance(x)
    return lv * torch.where(lr > ud, ud, lr)


def window_sum(t, k):
    """Non-overlapping k x k window sums of [B,1,H,W] -> [B,1,H/k,W/k]
    (the reference uses an all-ones Conv2d, attack.py:72-80)."""
    ones = torch.ones(1, 1, k, k, dtype=t.dtype)
    return torch.nn.functional.conv2d(t, ones, stride=k)


def struct_loss(adv_x, local_var_x):
    """attack.py:227-228."""
    mv = min_var_weighted_variance(adv_x).mean(1)
    return torch.mean(mv / (local_var_x + 1e-5), (1, 2))


def density_loss(mask, window):
    """attack.py:235 (unbiased variance of the window sums)."""
    return window_sum(mask, window).reshape(mask.shape[0], -1).var(1)


def group_lasso(mask, unit):
    """attack.py:243-244."""
    return unit * window_sum(mask ** 2, unit).sqrt().sum((1, 2, 3))


def patch_selection(mask, patch_budget, basic_unit=7):
    """attack.py:363-382 (selection='topk')."""
    gi = window_sum(mask, basic_unit)
    num_group = int(np.floor((mask.shape[2] * mask.shape[3] * patch_budget) / (basic_unit ** 2)))
    flat = gi.reshape(mask.shape[0], -1)
    val, idx = flat.topk(num_group)
    sel = torch.zeros_like(flat)
    for b in range(flat.shape[0]):
        sel[b, idx[b][val[b] > 0]] = 1
    sel = sel.reshape(gi.shape)
    return sel.repeat_interleave(basic_unit, dim=2).repeat_interleave(basic_unit, dim=3)


def collect_failure(model, adv_x1, y1, universe, targeted, batch_size):
    """attack.py:384-406 for ONE image [1,3,H,W]; returns sorted python list."""
    n_mask = universe.shape[0]
    failed = []
    with torch.no_grad():
        for j in range(int(np.ceil(n_mask / batch_size))):
            keep = universe[j * batch_size: min((j + 1) * batch_size, n_mask)]
            preds = model(occlude(adv_x1, keep)).argmax(-1)
            f = preds == y1
            if targeted:
                f = ~f
            failed.extend((f.nonzero().view(-1) + j * batch_size).tolist())
    return failed


def set_target(preds_adv, label):
    """attack.py:106-122 for one image: preds_adv [S], label python int.
    Returns (new_label, switched_to_targeted_criterion)."""
    wrong = preds_adv[preds_adv != label]
    if len(wrong) == 0:
        return label, False
    if len(wrong) > 1:
        return int(wrong.view(1, -1).mode(1)[0].item()), True
    return int(wrong[0].item()), True


# ----------------------------------------------------------------------------
# one hot-loop iteration: losses + gradients (attack.py:184-247)
# ----------------------------------------------------------------------------
def step_losses_and_grads(model, x, mask, pattern, y, idx, universe, crit_targeted, n_classes,
                          confidence, structured, density, coeff_group_lasso, stage, eps,
                          local_var_x, idx_dual=None, basic_unit=7, xforms=None):
    """x,pattern [B,3,H,W]; mask [B,1,H,W]; y [B] int64; idx [B,S] int (per-image
    mask indices); crit_targeted [B] bool; structured / coeff_group_lasso [B]
    python floats; returns a dict of tensors (all detached)."""
    B, _, H, W = x.shape
    S = idx.shape[1]
    mask = mask.detach().clone().requires_grad_(stage == 0)
    pattern = pattern.detach().clone().requires_grad_(True)
    delta = clip_paste(mask, pattern, x, eps)
    adv_x = x + delta
    keep = universe[torch.as_tensor(np.asarray(idx).reshape(-1))].reshape(B, S, 1, H, W)
    src = adv_x[:, None]
    if xforms is not None:                       # optional affine / colour EOT (not in the reference)
        from . import eot as _eot
        src = _eot.apply(adv_x, xforms)
    xm = occlude(src, keep)
    if idx_dual is not None:
        keep2 = universe[torch.as_tensor(np.asarray(idx_dual).reshape(-1))].reshape(B, S, 1, H, W)
        xm = occlude(xm, keep2)
    logits = model(xm.reshape(B * S, 3, H, W))
    ys = y[:, None].expand(B, S).reshape(-1)
    loss_adv = torch.stack([
        cw_loss(logits[b * S:(b + 1) * S], ys[b * S:(b + 1) * S], n_classes, bool(crit_targeted[b]), confidence)
        for b in range(B)])
    loss_struc = struct_loss(adv_x, local_var_x)
    loss = loss_adv.mean(1)
    st = torch.tensor([float(s) for s in structured], dtype=torch.float32)
    loss = loss + st * loss_struc * (st != 0)
    out = {}
    if stage == 0:
        loss_density = density_loss(mask, W // 8)
        if density != 0:
            loss = loss + density * loss_density
        gl = group_lasso(mask, basic_unit)
        loss = loss + torch.tensor([float(c) for c in coeff_group_lasso], dtype=torch.float32) * gl
        out["loss_density"] = loss_density.detach()
        out["group_lasso"] = gl.detach()
    loss.sum().backward()
    out.update(loss=loss.detach(), loss_adv=loss_adv.detach(), loss_struc=loss_struc.detach(),
               logits=logits.detach(), adv_x=adv_x.detach(), delta=delta.detach(),
               grad_pattern=pattern.grad.detach(),
               grad_mask=mask.grad.detach() if stage == 0 else None)
    return out


# ----------------------------------------------------------------------------
# full generate loop
# ----------------------------------------------------------------------------
class ImageState:
    """All scalar state the reference keeps in local variables, per image."""

    def __init__(self, lr, structured, y, targeted, rng):
        self.lr0 = np.float32(lr)
        self.coeff_group_lasso = 1e-5           # attack.py:87
        self.structured = structured
        self.y = int(y)
        self.targeted = bool(targeted)          # the 'targeted' variable (scan semantics)
        self.crit_targeted = bool(targeted)     # self.criterion.targeted (CW semantics)
        self.failed = []                        # attack.py:96
        self.certifiable = False
        self.rng = rng
        self.active = True
        self.reset_stage()

    def reset_stage(self):                      # attack.py:129-132
        self.lr = np.float32(self.lr0)
        self.loss_best = np.float32(np.inf)
        self.not_decay = 0
        self.num_failure = np.inf
        self.active = True


def sample_indices(st, i, n_mask, S):
    """attack.py:193-204 (one draw)."""
    n_ff = 0 if i < 1000 else min(len(st.failed), S // 2)
    parts = []
    if n_ff > 0:
        parts.append(st.rng.choice(st.failed, n_ff, replace=False))
    if S - n_ff > 0:
        parts.append(st.rng.choice(np.arange(n_mask), S - n_ff, replace=False))
    return np.concatenate(parts), n_ff


def bookkeeping(st, stage, i, loss_adv_s, idx, n_ff, loss_target):
    """attack.py:249-308 for one image.  Returns (save_best, stop_now)."""
    ok = (loss_adv_s < 1e-1)
    new_succ = idx[:n_ff][ok[:n_ff]]
    if len(new_succ) > 0:
        st.failed = np.setdiff1d(st.failed, new_succ).tolist()
    new_fail = idx[n_ff:][~ok[n_ff:]]
    if len(new_fail) > 0:
        st.failed = list(st.failed)
        st.failed.extend(new_fail)
        st.failed = np.unique(st.failed).tolist()
    success_all = bool(ok.all())
    st.certifiable = (len(st.failed) == 0)
    if len(st.failed) < st.num_failure:
        st.loss_best = np.float32(np.inf)
    certify_better = len(st.failed) <= st.num_failure
    loss_target = np.float32(loss_target)
    with np.errstate(invalid="ignore"):
        save_best = bool(certify_better and (np.float32(loss_target - st.loss_best) < np.float32(-1e-3)))
    if save_best:
        st.num_failure = len(st.failed)
        st.loss_best = loss_target
        st.not_decay = 0
    else:
        st.not_decay += 1
    early = st.not_decay > PATIENCE
    good = success_all and st.certifiable
    if stage == 0 and i > 200:
        st.coeff_group_lasso = st.coeff_group_lasso * SCALE_UP if good else st.coeff_group_lasso / SCALE_DOWN
    else:
        st.structured = st.structured * SCALE_UP if good else st.structured / SCALE_DOWN
    if early:
        st.lr = max(np.float32(st.lr * np.float32(0.1)), np.float32(.1 / 256.))
        st.not_decay = 0
    stop = bool(st.lr < np.float32(1e-3))
    return save_best, stop


def generate(model, x, patch_budget, n_classes, save_dir=None, batch_id=0, y=None, targeted=False,
             lr=1e-2, confidence=1e-1, clip_min=0, clip_max=1, max_iterations=5000, basic_unit=7,
             selection='topk', dropout=2, sampling_size=128, density=1e-3, structured=1e-3, eps=4.,
             dual=False, log=None, trace=None, **kwargs):
    """Restatement of DorPatch.generate (attack.py:51-361).  ``model`` maps
    [N,3,H,W] in [0,1] -> logits (torch CPU).  ``trace`` (a list) receives one
    dict per iteration for parity tests."""
    say = log if log is not None else (lambda s: None)
    B, _, H, W = x.shape
    adv_mask = torch.rand([B, 1, H, W])                      # attack.py:59 (CPU generator)
    adv_pattern = torch.rand(x.shape)                        # attack.py:60
    mask_best = torch.zeros_like(adv_mask)
    pattern_best = torch.zeros_like(adv_pattern)
    if y is None:
        with torch.no_grad():
            y = model(x).argmax(-1)
    # the reference builds two throw-away Conv2d modules here (attack.py:72-80);
    # their kaiming init consumes the CPU generator: 49 + window^2 draws.
    torch.nn.Conv2d(1, 1, basic_unit, stride=basic_unit, bias=False)
    torch.nn.Conv2d(1, 1, W // 8, stride=W // 8, bias=False)
    rects = omasks.universe_rects(W, dropout)
    universe = torch.from_numpy(omasks.rects_to_bool(rects, W))
    n_mask = universe.shape[0]
    S = min(sampling_size, n_mask)
    local_var_x = local_variance(x)[0].mean(1)               # attack.py:100
    if B == 1:
        rngs = [np.random]                                   # the global legacy stream, as the reference
    else:
        rngs = [np.random.RandomState(int(np.random.randint(0, 2 ** 31 - 1))) for _ in range(B)]
    states = [ImageState(lr, structured, y[b], targeted, rngs[b]) for b in range(B)]
    dir_0 = os.path.dirname(save_dir.rstrip('/')) if save_dir else None
    last_logits = None
    # Reference quirk (Q16): when stage 0 ends through the early-stop `break` (attack.py:310-315)
    # the break precedes `adv_pattern.grad.zero_()` (:342), so the gradient of that last stage-0
    # iteration is still in `.grad` and the first stage-1 backward accumulates onto it.
    stale_grad_pattern = torch.zeros_like(adv_pattern)

    for stage in range(2):
        say('============= Stage %d =============' % stage)
        for st in states:
            st.reset_stage()
        if stage == 0 and dir_0 and os.path.exists(os.path.join(dir_0, "adv_mask_%d.pt" % batch_id)):
            mask_best = torch.load(os.path.join(dir_0, "adv_mask_%d.pt" % batch_id))
            pattern_best = torch.load(os.path.join(dir_0, "adv_pattern_%d.pt" % batch_id))
            continue
        if stage == 1:
            with torch.no_grad():                            # attack.py:143-165
                adv_x = x + clip_paste(mask_best, pattern_best, x, eps)
                for b, st in enumerate(states):
                    if not st.targeted:
                        preds = model(adv_x[b:b + 1]).argmax(-1)
                        st.targeted = True
                        st.y, sw = set_target(preds, st.y)
                        st.crit_targeted = st.crit_targeted or sw
                pattern_best = adv_x.clone()
                torch.nn.Conv2d(1, 1, basic_unit, stride=basic_unit, bias=False)  # attack.py:365 RNG draw
                adv_mask = patch_selection(mask_best, patch_budget, basic_unit)
                mask_best = adv_mask.clone()
                adv_pattern = pattern_best.clone()
        adv_x = None
        for i in range(max_iterations):
            if stage == 0 and i == 500:                      # attack.py:169-182
                for b, st in enumerate(states):
                    if st.targeted or not st.active:
                        continue
                    st.targeted = True
                    preds = last_logits[b].argmax(-1)
                    y_new, sw = set_target(preds, st.y)
                    if y_new != st.y:
                        st.y = y_new
                        say(">> switch to targeted attack to category {:3d} at iteration: {:4d}".format(st.y, i))
                    st.crit_targeted = st.crit_targeted or sw
                    st.reset_stage()
                    st.failed = collect_failure(model, adv_x[b:b + 1], st.y, universe, st.targeted, S)
                    say(">> %d failures collected!" % len(st.failed))
            with torch.no_grad():
                adv_x = x + clip_paste(adv_mask, adv_pattern, x, eps)
            if i % 100 == 0:                                 # attack.py:187-190
                for b, st in enumerate(states):
                    if st.active:
                        st.failed = collect_failure(model, adv_x[b:b + 1], st.y, universe, st.targeted, S)
                        say(">> %d failures collected!" % len(st.failed))
            idx = np.zeros((B, S), dtype=np.int64)
            idx2 = np.zeros((B, S), dtype=np.int64) if dual else None
            nff = [0] * B
            for b, st in enumerate(states):
                if not st.active:
                    continue
                idx[b], nff[b] = sample_indices(st, i, n_mask, S)
                if dual:
                    idx2[b], _ = sample_indices(st, i, n_mask, S)
            yv = torch.tensor([st.y for st in states], dtype=torch.int64)
            r = step_losses_and_grads(
                model, x, adv_mask, adv_pattern, yv, idx, universe, [st.crit_targeted for st in states],
                n_classes, confidence, [st.structured for st in states], density,
                [st.coeff_group_lasso for st in states], stage, eps, local_var_x, idx2, basic_unit)
            if stage == 1 and i == 0:
                r["grad_pattern"] = stale_grad_pattern + r["grad_pattern"]
            last_logits = r["logits"].reshape(B, S, -1)
            loss_target = r["group_lasso"] if stage == 0 else r["loss_struc"]
            lr_used = np.zeros(B, dtype=np.float32)
            stop_flags = []
            for b, st in enumerate(states):
                if not st.active:
                    continue
                save_best, stop = bookkeeping(st, stage, i, r["loss_adv"][b].numpy(), idx[b], nff[b],
                                              loss_target[b].item())
                if save_best:
                    if stage == 0:
                        mask_best[b] = adv_mask[b]
                    pattern_best[b] = adv_pattern[b]
                if stop:
                    say("early stop at iteration: {:4d}".format(i))
                    if np.isinf(st.loss_best):
                        mask_best[b] = adv_mask[b]
                        pattern_best[b] = adv_pattern[b]
                    st.active = False
                    if stage == 0:
                        stale_grad_pattern[b] = r["grad_pattern"][b]
                else:
                    lr_used[b] = st.lr
                stop_flags.append(stop)
            if trace is not None:
                trace.append(dict(stage=stage, i=i, idx=idx.copy(), loss_adv=r["loss_adv"].numpy().copy(),
                                  loss_struc=r["loss_struc"].numpy().copy(),
                                  group_lasso=r["group_lasso"].numpy().copy() if stage == 0 else None,
                                  lr=lr_used.copy(), structured=[st.structured for st in states],
                                  coeff=[st.coeff_group_lasso for st in states],
                                  n_failed=[len(st.failed) for st in states]))
            if i % 20 == 0 and any(st.active for st in states):   # attack.py:317-330
                preds = r["logits"].argmax(-1)
                ys = yv[:, None].expand(B, S).reshape(-1)
                acc = (preds == ys).sum().item() / (B * S) * 100
                l2 = torch.sqrt((r["delta"] ** 2).sum((1, 2, 3)))
                s = "iteration: {:4d}, accuracy: {:.2f}, loss: {:.2f}, adv: {:.2f}, l2 norm: {:.2f}, structural: {:.2f}".format(
                    i, acc, r["loss"].mean().item(), r["loss_adv"].mean().item(), l2.mean().item(),
                    r["loss_struc"].mean().item())
                if stage == 0:
                    s += ", group lasso: {:.2f}, density: {:.2f}".format(
                        r["group_lasso"].mean().item(), r["loss_density"].mean().item())
                say(s)
            if not any(st.active for st in states):
                break
            with torch.no_grad():                            # attack.py:332-342
                lrv = torch.from_numpy(lr_used)[:, None, None, None]
                if stage == 0:
                    adv_mask = (adv_mask - lrv * r["grad_mask"].sign()).clamp(clip_min, clip_max)
                adv_pattern = (adv_pattern - lrv * r["grad_pattern"].sign()).clamp(clip_min, clip_max)
        for b, st in enumerate(states):                      # attack.py:344-346
            if np.isinf(st.loss_best) and st.active:
                mask_best[b] = adv_mask[b]
                pattern_best[b] = adv_pattern[b]
        if stage == 0:
            if dir_0:
                os.makedirs(dir_0, exist_ok=True)
                torch.save(mask_best, os.path.join(dir_0, "adv_mask_%d.pt" % batch_id))
                torch.save(pattern_best, os.path.join(dir_0, "adv_pattern_%d.pt" % batch_id))
            for b, st in enumerate(states):                  # attack.py:357-359 (arity fixed)
                if not st.targeted and last_logits is not None:
                    st.y, sw = set_target(last_logits[b].argmax(-1), st.y)
                    st.crit_targeted = st.crit_targeted or sw
    return mask_best, pattern_best
