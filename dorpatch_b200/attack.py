"""DorPatch patch generation on the native H100 engine -- host control flow.

Drop-in for reference attack.py: ``DorPatch().generate(...)`` keeps the reference's
signature (attack.py:51-53), side effects (prints, stage-0 artefacts in the parent directory,
RNG consumption) and return value.  Everything numeric in the hot loop (attack.py:184-247,
332-342) runs in libdorpatch.so through ``dorpatch_b200.engine.Engine``; what stays here is
the scalar state machine of attack.py:249-330 (failed-mask set, best snapshot, patience / lr
decay, coefficient adaptation) and the numpy sampling of attack.py:193-204, both of which
depend on the legacy global numpy RNG and Python-float arithmetic and are O(S) per step.

Semantics beyond the reference (see DESIGN.md):
  * B > 1 runs B independent single-image problems side by side (the reference is
    batch-size-1 only); all scalar state is per image.  B == 1 reproduces the reference's
    control flow and RNG stream exactly.
  * the two ``set_target(preds_adv)`` call sites with a missing argument (attack.py:155,359,
    a TypeError in the reference) pass the label.
  * EOT sharding: with torch.distributed initialised, each rank evaluates S/world samples and
    the ranks all-reduce the patch gradient once per step; the periodic universe scan
    (collect_failure) is split over the ranks by distinct occlusion and its fail bits all-gathered.
    PatchCleanser evaluation shards its masked forwards with the same split (shard_range, sharded_predict,
    sharded_checks).
  * ``pc_n_patch=2`` draws the universe from the two-patch PatchCleanser window (the reference
    always uses the one-patch window, attack.py:25-31); the universe scans forward each distinct
    occlusion once.
  * ``eot_sampler="device"`` draws the EOT occlusions on the GPU (dp_eot_draw): the rule of attack.py:193-218 from a
    counter-based generator seeded per image, so the draws are reproducible but not numpy's; indices, rectangles and the
    failed-set update never leave the device.
  * ``checkpoint=<path>`` saves everything the loop carries from one step to the next every ``checkpoint_every`` steps
    and at each stage boundary; a later call with the same arguments continues from the file as the uninterrupted call
    would have (the reference resumes only at the stage-0 cache and main.py's per-batch artefacts).
"""
import hashlib
import io
import os
import sys
import tempfile

import numpy as np
import torch

from . import masks as _masks
from .utils import unwrap_native

PATIENCE = 200
SCALE_UP = 1.2
SCALE_DOWN = np.sqrt(SCALE_UP ** 3)


# ----------------------------------------------------------------------------------------
# public helpers kept for API compatibility with the reference module
# ----------------------------------------------------------------------------------------
class CW_loss():
    """attack.py:10-23 (torch ops; the hot loop uses the fused native K4 kernel instead)."""

    def __init__(self, num_classes, targeted=False, confidence=0):
        self.num_classes, self.targeted, self.confidence = num_classes, targeted, confidence

    def __call__(self, logits, y):
        idx = torch.arange(logits.shape[0], device=logits.device)
        real = logits[idx, y]
        masked = logits.clone()
        masked[idx, y] = -1e4
        other = masked.max(1)[0]
        margin = (other - real) if self.targeted else (real - other)
        return torch.clamp(self.confidence + margin, min=0.)


def get_mask_set(img_size, dropout_size, dropout):
    """attack.py:25-31; returns the bool mask tensor like the reference (API compatibility)."""
    from .defenses.PatchCleanser import MaskWindow
    mw = MaskWindow(img_size, dropout_size)
    return mw.mask_set if dropout == 1 else (mw.double_mask_set if dropout == 2 else None)


def local_variance(x):
    """attack.py:33-39 incl. its raw last row / column (values only)."""
    lr = torch.cat([(x[..., :, :-1] - x[..., :, 1:]).abs(), x[..., :, -1:]], dim=-1)
    ud = torch.cat([(x[..., :-1, :] - x[..., 1:, :]).abs(), x[..., -1:, :]], dim=-2)
    return lr + ud, lr, ud


def min_var_weighted_variance(x):
    """attack.py:41-45 (values only)."""
    lv, lr, ud = local_variance(x)
    return lv * torch.minimum(lr, ud)


# ----------------------------------------------------------------------------------------
class _ImageState(object):
    """The scalars the reference keeps in local variables, for one image."""

    def __init__(self, lr, structured, y, targeted, rng):
        self.lr0 = np.float32(lr)
        self.coeff_group_lasso = 1e-5            # attack.py:87
        self.structured = structured
        self.y = int(y)
        self.targeted = bool(targeted)           # the `targeted` variable (scan semantics)
        self.crit_targeted = bool(targeted)      # self.criterion.targeted
        self.failed = []                         # host copy of the failed-mask set (authoritative only when dev is None)
        self.n_failed = 0
        self.dev = None                          # (engine, image slot): the set lives on the device as a bitmap (N2)
        self.certifiable = False
        self.rng = rng
        self.reset()

    def set_failed(self, indices):               # a universe scan replaced the set (attack.py:187-190)
        self.failed = list(indices)
        self.n_failed = len(self.failed)
        if self.dev is not None:
            self.dev[0].failed_write(self.dev[1], self.failed)

    def reset(self):                             # attack.py:129-132
        self.lr = np.float32(self.lr0)
        self.loss_best = np.float32(np.inf)
        self.not_decay = 0
        self.num_failure = np.inf
        self.active = True

    def sample(self, i, n_mask, S):              # attack.py:193-204
        n_ff = 0 if i < 1000 else min(self.n_failed, S // 2)
        parts = []
        if n_ff > 0:
            if self.dev is not None:             # the only reader of the set's CONTENT: fetch the sorted indices
                self.failed = self.dev[0].failed_read(self.dev[1])
            parts.append(self.rng.choice(self.failed, n_ff, replace=False))
        if S - n_ff > 0:
            parts.append(self.rng.choice(np.arange(n_mask), S - n_ff, replace=False))
        return np.concatenate(parts), n_ff

    def bookkeeping(self, stage, i, loss_adv, idx, n_ff, loss_target, n_failed=None):   # attack.py:249-308
        """n_failed: size of the failed set after this step when the device keeps it (dp_failed_set_update);
        None = update the host list here (attack.py:259-267)."""
        ok = loss_adv < np.float32(1e-1)
        if n_failed is None:
            gone = idx[:n_ff][ok[:n_ff]]
            if len(gone) > 0:
                self.failed = np.setdiff1d(self.failed, gone).tolist()
            new = idx[n_ff:][~ok[n_ff:]]
            if len(new) > 0:
                self.failed = np.unique(list(self.failed) + list(new)).tolist()
            n_failed = len(self.failed)
        self.n_failed = int(n_failed)
        self.certifiable = n_failed == 0
        if n_failed < self.num_failure:
            self.loss_best = np.float32(np.inf)
        loss_target = np.float32(loss_target)
        with np.errstate(invalid="ignore"):
            improved = bool(n_failed <= self.num_failure and
                            np.float32(loss_target - self.loss_best) < np.float32(-1e-3))
        if improved:
            self.num_failure, self.loss_best, self.not_decay = n_failed, loss_target, 0
        else:
            self.not_decay += 1
        plateau = self.not_decay > PATIENCE
        good = bool(ok.all()) and self.certifiable
        if stage == 0 and i > 200:
            self.coeff_group_lasso = self.coeff_group_lasso * SCALE_UP if good else self.coeff_group_lasso / SCALE_DOWN
        else:
            self.structured = self.structured * SCALE_UP if good else self.structured / SCALE_DOWN
        if plateau:
            self.lr = max(np.float32(self.lr * np.float32(0.1)), np.float32(.1 / 256.))
            self.not_decay = 0
        return improved, bool(self.lr < np.float32(1e-3))

    def state(self):
        """Everything generate() carries from one step to the next for this image, as plain values (a checkpoint's)."""
        failed = self.dev[0].failed_read(self.dev[1]) if self.dev is not None else self.failed
        return dict(lr=float(self.lr), loss_best=float(self.loss_best), not_decay=int(self.not_decay),
                    num_failure=float(self.num_failure) if np.isinf(self.num_failure) else int(self.num_failure),
                    coeff_group_lasso=float(self.coeff_group_lasso), structured=float(self.structured), y=int(self.y),
                    targeted=bool(self.targeted), crit_targeted=bool(self.crit_targeted),
                    certifiable=bool(self.certifiable), active=bool(self.active), n_failed=int(self.n_failed),
                    failed=torch.tensor(np.asarray(failed, np.int32).reshape(-1)))

    def load_state(self, d):
        """Inverse of state(): the failed set goes back to the device when it lives there."""
        self.set_failed(d["failed"].tolist())
        self.lr, self.loss_best = np.float32(d["lr"]), np.float32(d["loss_best"])
        for k in ("not_decay", "num_failure", "coeff_group_lasso", "structured", "y", "targeted", "crit_targeted",
                  "certifiable", "active", "n_failed"):
            setattr(self, k, d[k])


def _may_prefetch(states, i, max_iterations):
    """May step i+1's samples be drawn before step i's bookkeeping without changing the reference's RNG consumption?
    Yes iff the stage does run an iteration i+1 with the same set of active images and the draw reads nothing step i
    writes: i+1 < 1000 (no samples from the failed set, attack.py:193-198), i+1 < max_iterations, and no active image can
    stop at step i -- a stop (attack.py:306-315) needs a plateau (not_decay > PATIENCE after the step, so >= PATIENCE - 1
    before it, conservatively) whose decayed lr falls below 1e-3 (10 % margin on the float comparison)."""
    if i + 1 >= max_iterations or i + 1 >= 1000:
        return False
    return not any(s.active and s.not_decay >= PATIENCE - 1 and float(s.lr) * 0.1 < 1.1e-3 for s in states)


def _pick_target(preds, label):
    """attack.py:106-122 for one image; returns (label, switched)."""
    preds = np.asarray(preds).reshape(-1)
    wrong = preds[preds != label]
    if wrong.size == 0:
        return label, False
    if wrong.size > 1:
        vals, counts = np.unique(wrong, return_counts=True)     # torch.mode: smallest of the most frequent
        return int(vals[np.argmax(counts)]), True
    return int(wrong[0]), True


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 \
            and os.environ.get("DORPATCH_SHARD", "eot") == "eot":
        return dist
    return None


def _assert_same_on_all_ranks(dist, arr, device, what,
                              hint="seed every rank identically (utils.set_random_seed) before generate()"):
    """Cheap consistency check of host-side state that EOT sharding assumes identical on every rank."""
    a = np.ascontiguousarray(arr).astype(np.int64).ravel()
    chk = torch.tensor([int(a.sum()), int((a * (np.arange(a.size) % 8191 + 1)).sum())], dtype=torch.int64, device=device)
    lo, hi = chk.clone(), chk.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    if not torch.equal(lo, hi):
        raise RuntimeError("ranks disagree on %s: %s" % (what, hint))


def exchange_shards(dist, G, loss_adv, preds, defer=False):
    """The only cross-rank exchange of a step: SUM all-reduce of the patch gradient G
    [B,3,H,W] (each rank holds the sum over ITS S/world samples, already divided by the global
    S) and an all-gather of the per-sample results [B,S/world] -> [B,S] in rank order, so every
    rank takes the identical bookkeeping decisions and the identical sign step.

    Order matters for overlap: both collectives run on the process group's one NCCL stream, so the tiny
    all-gather goes FIRST and its single device->host copy waits for it alone; the large all-reduce
    (B*0.6 MB) is enqueued behind it asynchronously and runs under the host bookkeeping.  With
    ``defer=True`` the all-reduce's work handle is returned as a third value and the caller waits on it
    right before the sign step (``work.wait()`` orders the compute stream after NCCL's; it does not block
    the host); otherwise the wait happens here."""
    world = dist.get_world_size()
    s_loc = loss_adv.shape[1]
    pack = torch.from_numpy(np.concatenate([loss_adv, preds.astype(np.float32)], 1))
    if G.is_cuda:
        pack = pack.pin_memory().to(G.device, non_blocking=True)
        allp = torch.empty((world,) + tuple(pack.shape), dtype=pack.dtype, device=G.device)
        dist.all_gather_into_tensor(allp, pack)
        work = dist.all_reduce(G, async_op=True)
        allp = allp.cpu()                                   # one D2H + one synchronisation for all ranks' results
    else:                                                   # gloo (CPU tests)
        outs = [torch.empty_like(pack) for _ in range(world)]
        dist.all_gather(outs, pack)
        work = dist.all_reduce(G, async_op=True)
        allp = torch.stack(outs)
    allp = allp.numpy()
    loss_all = np.concatenate([allp[r][:, :s_loc] for r in range(world)], 1)
    preds_all = np.concatenate([allp[r][:, s_loc:] for r in range(world)], 1).astype(np.int32)
    if defer:
        return loss_all, preds_all, work
    work.wait()
    return loss_all, preds_all


def shard_range(n, rank, world, unit=1):
    """The contiguous shard [lo, hi) of n items that `rank` of `world` takes: ceil(units / world) whole units of `unit`
    items each, in rank order, the last unit keeping its length.  Every item lands in exactly one shard, cuts fall at
    multiples of `unit` only, and a rank past the last unit gets an empty shard.  The one sharding convention of the
    universe scan (unit 1) and of PatchCleanser's masked forwards (unit = the engine's chunk)."""
    units = -(-n // unit)
    per = -(-units // world) * unit
    return min(rank * per, n), min((rank + 1) * per, n)


def _all_gather_rows(dist, row, device):
    """All-gather one equally long 1-D tensor per rank -> numpy [world, len] in rank order, on every rank."""
    row = row.to(device)
    outs = [torch.empty_like(row) for _ in range(dist.get_world_size())]
    dist.all_gather(outs, row)
    return torch.stack(outs).cpu().numpy()


def collective_device(dist):
    """Where the tensors of a collective live: the current GPU under NCCL, else the host (gloo)."""
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")


def sharded_predict(predict, n, chunk, dist=None):
    """The int32 labels of one forward call over n samples that the engine runs in chunks of `chunk`:
    `predict(lo, hi)` forwards samples [lo, hi) of the call as one call.  Without dist this is predict(0, n), the single
    call.  With torch.distributed every rank forwards its shard_range in whole chunks, so each of its chunks holds the
    samples of one chunk of the single call and gives the same logits (the engine computes a sample from its chunk
    alone, DESIGN section 5); the labels are all-gathered in rank order and every rank returns the single call's array.
    A rank with an empty shard forwards nothing and still joins the all-gather."""
    if dist is None:
        return np.asarray(predict(0, n), dtype=np.int32)
    rank, world = dist.get_rank(), dist.get_world_size()
    per = shard_range(n, 0, world, chunk)[1]
    lo, hi = shard_range(n, rank, world, chunk)
    mine = torch.zeros(per, dtype=torch.int32)
    if hi > lo:
        mine[:hi - lo] = torch.from_numpy(np.asarray(predict(lo, hi), dtype=np.int32))
    return np.ascontiguousarray(_all_gather_rows(dist, mine, collective_device(dist)).reshape(-1)[:n])


def sharded_checks(check, m, dist=None):
    """[check(i) for i in range(m)] as bools, each check a whole call: without dist all of them in order on this rank;
    with torch.distributed check i runs on rank i % world (round-robin in the given order) and the results are
    all-gathered, so every rank returns the same list, in the same order.  m must be the same on every rank."""
    if dist is None or m == 0:
        return [bool(check(i)) for i in range(m)]
    rank, world = dist.get_rank(), dist.get_world_size()
    mine = torch.zeros(-(-m // world), dtype=torch.uint8)
    for j, i in enumerate(range(rank, m, world)):
        mine[j] = bool(check(i))
    rows = _all_gather_rows(dist, mine, collective_device(dist))
    return [bool(rows[i % world, i // world]) for i in range(m)]


def scan_failures(predict, all_rects, y, targeted, dist=None, device="cpu", inv=None):
    """collect_failure for one image (attack.py:384-406): indices of the universe masks under
    which the attack fails.  `predict(rects[k,4,4]) -> labels[k]`.  With torch.distributed the
    universe is split into contiguous shards, one per rank (SURVEY section 8e: the scan is
    embarrassingly parallel over the mask index), and the fail bits are all-gathered, so every
    rank returns the identical list and takes the identical bookkeeping decisions.
    With `inv`, all_rects holds the universe's distinct occlusions (masks.distinct_occlusions) and
    universe mask k is all_rects[inv[k]]: each occlusion is forwarded once (on one rank) and its
    result spread to every index sharing it, so the list is the one the full scan returns."""
    n = all_rects.shape[0]
    if dist is None:
        f = np.asarray(predict(all_rects)) == y
    else:
        rank, world = dist.get_rank(), dist.get_world_size()
        per = shard_range(n, 0, world)[1]
        lo, hi = shard_range(n, rank, world)
        bits = torch.zeros(per, dtype=torch.uint8)
        if hi > lo:
            bits[:hi - lo] = torch.from_numpy((np.asarray(predict(all_rects[lo:hi])) == y).astype(np.uint8))
        f = _all_gather_rows(dist, bits, device).reshape(-1)[:n].astype(bool)
    if inv is not None:
        f = f[inv]
    if targeted:
        f = ~f
    return np.nonzero(f)[0].tolist()


# ----------------------------------------------------------------------------------------
# step-level checkpoints of generate()
CHECKPOINT_VERSION = 1


def checkpoint_fingerprint(x, y, world, precision, **kw):
    """What a checkpoint must have been written by: the image batch (shape and a content hash), the effective labels,
    every keyword that changes the computation (`kw`, in a fixed order), the world size and the engine precision.
    A list of (field, value) pairs of plain Python values, so the first differing field can be named."""
    xb = x.detach().float().contiguous().cpu().numpy()
    fp = [("x_shape", list(xb.shape)), ("x_sha256", hashlib.sha256(xb.tobytes()).hexdigest()),
          ("y", [int(v) for v in y])]
    for k in sorted(kw):
        v = kw[k]
        if isinstance(v, (list, tuple, np.ndarray)):
            v = [int(s) for s in v]
        elif isinstance(v, (bool, np.bool_)):
            v = bool(v)
        elif isinstance(v, (int, np.integer)):
            v = int(v)
        elif isinstance(v, (float, np.floating)):
            v = float(v)
        fp.append((k, v))
    fp += [("world_size", int(world)), ("precision", str(precision))]
    return fp


def rng_state_out(rs):
    """A numpy RandomState's (or the legacy global stream's) state as values torch.load(weights_only=True) reads back."""
    name, keys, pos, has_gauss, cached = rs.get_state()
    return [name, torch.from_numpy(keys.astype(np.int64)), int(pos), int(has_gauss), float(cached)]


def rng_state_in(rs, state):
    name, keys, pos, has_gauss, cached = state
    rs.set_state((name, keys.numpy().astype(np.uint32), pos, has_gauss, cached))


def save_checkpoint(path, ckpt):
    """Replace `path` by `ckpt` atomically: write a temporary file in the same directory, flush and fsync it, then
    os.replace it over the old one, so a process killed mid-write leaves the previous checkpoint intact."""
    d = os.path.dirname(os.path.abspath(path))
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(path) + ".", suffix=".tmp", dir=d)
    try:
        with os.fdopen(fd, "wb") as f:
            torch.save(ckpt, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    dfd = os.open(d, os.O_RDONLY)                            # make the rename itself durable
    try:
        os.fsync(dfd)
    finally:
        os.close(dfd)


def load_checkpoint(path, fingerprint):
    """Read a checkpoint written by save_checkpoint and check that it belongs to the call whose fingerprint is given:
    ValueError naming the format version or the first field that differs.  Returns (checkpoint, digest of the file's
    bytes as uint16 words)."""
    with open(path, "rb") as f:
        raw = f.read()
    ck = torch.load(io.BytesIO(raw), map_location="cpu", weights_only=True)
    if not isinstance(ck, dict) or ck.get("version") != CHECKPOINT_VERSION:
        raise ValueError("checkpoint %s: format version %r, this code reads version %d"
                         % (path, ck.get("version") if isinstance(ck, dict) else None, CHECKPOINT_VERSION))
    saved = dict((k, v) for k, v in ck["fingerprint"])
    for k, v in fingerprint:
        if k not in saved or saved[k] != v:
            raise ValueError("checkpoint %s was written by a different call: %s differs (checkpoint: %r, this call: %r)"
                             % (path, k, saved.get(k, "<missing>"), v))
    if len(saved) != len(fingerprint):
        extra = sorted(set(saved) - set(k for k, _ in fingerprint))
        raise ValueError("checkpoint %s was written by a different call: %s differs" % (path, extra[0]))
    return ck, np.frombuffer(hashlib.sha256(raw).digest(), np.uint16)


_SHARED = "every rank must read the same checkpoint file: keep it in a directory all ranks share"


def read_checkpoint(path, fingerprint, dist=None, device="cpu"):
    """The validated checkpoint at `path`, or None if there is none.  Under torch.distributed every rank reads the file
    and the ranks check that they agree on whether it exists and on its contents."""
    exists = os.path.exists(path)
    if dist:
        _assert_same_on_all_ranks(dist, [int(exists)], device, "whether %s exists" % path, _SHARED)
    if not exists:
        return None
    ck, digest = load_checkpoint(path, fingerprint)
    if dist:
        _assert_same_on_all_ranks(dist, digest, device, "the contents of %s" % path, _SHARED)
    return ck


def write_checkpoint(path, make, dist=None):
    """save_checkpoint(path, make()) on rank 0 alone (every rank holds the same state); the other ranks wait at a barrier
    until the file is in place."""
    if dist is None or dist.get_rank() == 0:
        save_checkpoint(path, make())
    if dist:
        dist.barrier()


def remove_checkpoint(path, dist=None):
    """Delete the checkpoint of a finished call (rank 0), so that a later call with the same path starts fresh."""
    if (dist is None or dist.get_rank() == 0) and os.path.exists(path):
        os.remove(path)
    if dist:
        dist.barrier()


class DorPatch(object):
    def __init__(self):
        self.last_stats = {}

    # ------------------------------------------------------------------------------------
    def generate(self, model, x, patch_budget, n_classes, save_dir, batch_id, y=None, targeted=False,
                 lr=1e-2, confidence=1e-1, clip_min=0, clip_max=1, max_iterations=5000, basic_unit=7,
                 selection='topk', dropout=2, sampling_size=128, density=1e-3, structured=1e-3, eps=4., dual=False,
                 eot_affine=0.0, eot_colour=0.0, eot_seed=0, pc_n_patch=1, eot_sampler="host", checkpoint=None,
                 checkpoint_every=100, **kwargs):
        """Reference signature (attack.py:51-53) plus three opt-in keywords for the affine / colour
        EOT extension (default 0 = off = the reference's behaviour).  `image_seeds=[s_0..s_{B-1}]` (keyword)
        makes row b of a B > 1 call replay the B == 1 run seeded with s_b (SURVEY section 0: parity of the
        batched configs is defined per image against a B == 1 reference run).
        `pc_n_patch=2` trains against the two-patch PatchCleanser: the EOT occlusions and the universe scans come from
        MaskWindow(W, r, 2) (dropout 1: its 630 pairs per ratio; dropout 2: its 22 680 three-rectangle masks per ratio)
        instead of the reference's one-patch window (1, the default).
        `eot_sampler="device"` draws every step's EOT occlusions on the GPU (dp_eot_draw) instead of with numpy on the
        host (`"host"`, the default and the reference's stream): the indices, their rectangles and the failed-set update
        stay on the device, so a long run is paced by the GPU.  The draws are reproducible from per-image seeds --
        `image_seeds[b]`, else B seeds drawn once from the global numpy stream -- but are not numpy's.
        `checkpoint=<path>` makes the call resumable: if the file exists, the call continues from the step it records
        (ValueError if it was written by a call with other inputs, keywords, world size or precision); while running it
        rewrites the file atomically after every `checkpoint_every`-th step of a stage and at the stage boundary, and
        deletes it on return.  The resumed call returns, prints from the resumed step on, and leaves the global numpy
        and torch RNG states as the uninterrupted call would have (bit for bit with the fp32 engine, or with any
        precision under DORPATCH_AUTOTUNE=0, without affine / colour EOT).  None (the default) reads and writes nothing."""
        if checkpoint is not None and (isinstance(checkpoint_every, bool) or
                                       not isinstance(checkpoint_every, (int, np.integer)) or checkpoint_every < 1):
            raise ValueError("checkpoint_every=%r must be a positive integer" % (checkpoint_every,))
        if eot_sampler not in ("host", "device"):
            raise ValueError("eot_sampler=%r: 'host' or 'device'" % (eot_sampler,))
        on_device = eot_sampler == "device"
        if on_device and os.environ.get("DORPATCH_FAILED", "device") == "host":
            raise ValueError("eot_sampler='device' samples from the failed sets on the device; DORPATCH_FAILED=host keeps "
                             "them on the host")
        W = x.shape[-1]
        if isinstance(basic_unit, bool) or not isinstance(basic_unit, (int, np.integer)) or basic_unit < 1 \
                or W % basic_unit != 0:
            # the reference fails later on such a unit, at stage 1's clip broadcast
            raise ValueError("basic_unit=%r must be a positive integer dividing the image size %d" % (basic_unit, W))
        basic_unit = int(basic_unit)
        if selection != 'topk':
            raise NotImplementedError("selection=%r" % (selection,))
        if dropout not in (1, 2):
            raise NotImplementedError("dropout=%r (the reference's dropout=0 path is degenerate)" % (dropout,))
        if pc_n_patch not in (1, 2):
            raise NotImplementedError("pc_n_patch=%r: PatchCleanser masks exist for 1 or 2 patches" % (pc_n_patch,))
        if dual and pc_n_patch == 2 and dropout == 2:
            raise NotImplementedError("dual=True with pc_n_patch=2, dropout=2 needs 6 rectangles per sample; "
                                      "the native kernels take 4")
        net = unwrap_native(model)
        if not x.is_cuda:
            raise RuntimeError("DorPatch.generate needs CUDA tensors: the hot loop exists only as native sm_90a kernels")
        x = x.contiguous().float()
        B, _, H, W = x.shape
        eng = net.engine(W, max_images=B)
        dev = x.device
        dist = _dist()
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist else (0, 1)

        image_seeds = kwargs.get("image_seeds")
        if image_seeds is not None and len(image_seeds) != B:
            raise ValueError("image_seeds needs one seed per image")
        if image_seeds is None:
            adv_mask = torch.rand([B, 1, H, W]).to(dev)          # attack.py:59 (CPU generator)
            adv_pattern = torch.rand(x.shape).to(dev)            # attack.py:60
        else:
            # row b reproduces a B == 1 run preceded by utils.set_random_seed(image_seeds[b]): its own torch-CPU
            # generator for the two initial draws and its own legacy numpy stream for the mask sampling
            gens = [torch.Generator().manual_seed(int(s)) for s in image_seeds]
            mp = [(torch.rand([1, 1, H, W], generator=g), torch.rand([1, 3, H, W], generator=g)) for g in gens]
            adv_mask = torch.cat([m for m, _ in mp]).to(dev)
            adv_pattern = torch.cat([q for _, q in mp]).to(dev)
        if dist:
            # EOT sharding needs bit-identical patch state on every rank: rank 0's draw is authoritative
            dist.broadcast(adv_mask, 0)
            dist.broadcast(adv_pattern, 0)
        mask_best = torch.zeros_like(adv_mask)
        pattern_best = torch.zeros_like(adv_pattern)
        if y is None:                                            # attack.py:67-69
            y = torch.from_numpy(eng.predict(x).astype(np.int64))
        y = [int(v) for v in (y.tolist() if torch.is_tensor(y) else y)]
        # the reference constructs two throw-away Conv2d modules whose kaiming init draws
        # 49 + (W/8)^2 values from the CPU generator (attack.py:72-80)
        torch.nn.Conv2d(1, 1, basic_unit, stride=basic_unit, bias=False)
        torch.nn.Conv2d(1, 1, W // 8, stride=W // 8, bias=False)

        table = _masks.universe(W, dropout, pc_n_patch)          # attack.py:83-85 as rectangles
        n_mask = table.shape[0]
        S = min(sampling_size, n_mask)
        if S % world != 0:
            raise ValueError("sampling_size=%d must be divisible by the world size %d" % (S, world))
        S_loc = S // world
        distinct, inv = _masks.distinct_occlusions(table, len(_masks.DROPOUT_SIZES))   # scans forward each once
        scan_rects = _masks.gather(distinct, np.arange(len(distinct)))

        if on_device:                                            # the draws' per-image seeds; no host stream
            seeds = [int(s) for s in image_seeds] if image_seeds is not None else \
                [int(np.random.randint(0, 2 ** 31 - 1)) for _ in range(B)]
            rngs = [None] * B
        elif image_seeds is not None:
            rngs = [np.random.RandomState(int(s)) for s in image_seeds]
        elif B == 1:
            rngs = [np.random]                                   # the global legacy stream, as the reference
        else:
            rngs = [np.random.RandomState(int(np.random.randint(0, 2 ** 31 - 1))) for _ in range(B)]
        st = [_ImageState(lr, structured, y[b], targeted, rngs[b]) for b in range(B)]
        device_sets = os.environ.get("DORPATCH_FAILED", "device") != "host"
        if device_sets:                                          # failed-mask sets as device bitmaps (SURVEY 8f N2)
            eng.failed_reset(n_mask)
            for b, s in enumerate(st):
                s.dev = (eng, b)
                s.set_failed([])
        if on_device:
            eng.eot_universe(table)
        dir_0 = os.path.dirname(save_dir.rstrip('/')) if save_dir else None
        G = torch.zeros_like(x)
        use_eot = (eot_affine != 0.0) or (eot_colour != 0.0)
        eot_rng = np.random.RandomState(eot_seed)
        # Reference quirk: an early-stop `break` in stage 0 (attack.py:310-315) skips
        # `adv_pattern.grad.zero_()` (:342), so the first stage-1 backward accumulates onto the
        # gradient of the last stage-0 iteration.  Kept per image, zero unless stage 0 stopped early.
        stale_gp = torch.zeros_like(x)
        have_stale = False
        last_preds = None
        steps = 0
        scans = [0, 0]                                           # universe scans, dp_predict forwards they issued here

        def scan(b, adv_x):                                      # collect_failure, attack.py:384-406
            def predict(r):
                scans[1] += r.shape[0]
                return eng.predict(adv_x[b:b + 1], r.shape[0], r)
            # distinct occlusions split over the ranks (if any), the result expanded to every universe index
            failed = scan_failures(predict, scan_rects, st[b].y, st[b].targeted, dist, dev, inv=inv)
            scans[0] += 1
            print(">> %d failures collected!" % len(failed))
            return failed

        def draw(i):                                             # attack.py:193-204 (+ :208-218 dual) for every active image
            if on_device:                                        # indices and rectangles stay on the device
                got = eng.eot_draw(seeds, stage, i, [s.active for s in st], S, dual, rank, world,
                                   host=bool(dist) and i % 100 == 0)
                return (got[0] if got else None), None, None, None
            idx = np.zeros((B, S), np.int64)
            idx2 = np.zeros((B, S), np.int64) if dual else None
            nff = [0] * B
            for b, s in enumerate(st):
                if s.active:
                    idx[b], nff[b] = s.sample(i, n_mask, S)
                    if dual:
                        idx2[b], _ = s.sample(i, n_mask, S)
            sl = slice(rank * S_loc, (rank + 1) * S_loc)
            return idx, idx2, nff, _masks.gather(table, idx[:, sl], idx2[:, sl] if dual else None)

        start_stage, start_i = 0, 0
        adv_x_prev = None
        if checkpoint is not None:
            fingerprint = checkpoint_fingerprint(
                x, y, world, eng.precision, patch_budget=patch_budget, targeted=targeted, lr=lr, confidence=confidence,
                clip_min=clip_min, clip_max=clip_max, max_iterations=max_iterations, basic_unit=basic_unit,
                selection=selection, dropout=dropout, sampling_size=sampling_size, density=density,
                structured=structured, eps=eps, dual=dual, eot_affine=eot_affine, eot_colour=eot_colour,
                eot_seed=eot_seed, pc_n_patch=pc_n_patch, eot_sampler=eot_sampler, image_seeds=image_seeds)
            ck = read_checkpoint(checkpoint, fingerprint, dist, dev)
            if ck is not None:
                # the set-up above drew from the RNG streams as a fresh call does; the checkpoint's states replace them
                cs = ck["state"]
                start_stage, start_i = int(ck["stage"]), int(ck["i"])
                for s, d in zip(st, cs["images"]):
                    s.load_state(d)
                adv_mask, adv_pattern = cs["adv_mask"].to(dev), cs["adv_pattern"].to(dev)
                mask_best, pattern_best = cs["mask_best"].to(dev), cs["pattern_best"].to(dev)
                have_stale = cs["have_stale"]
                if have_stale:
                    stale_gp = cs["stale_gp"].to(dev)
                last_preds = None if cs["last_preds"] is None else cs["last_preds"].numpy()
                adv_x_prev = None if cs["adv_x_prev"] is None else cs["adv_x_prev"].to(dev)
                steps = cs["steps"]
                scans[:] = cs["scans"]
                if on_device:
                    seeds[:] = cs["seeds"]
                for r, rs in zip(rngs, cs["rngs"]):
                    if rs is not None:
                        rng_state_in(r, rs)
                rng_state_in(eot_rng, cs["eot_rng"])
                rng_state_in(np.random, cs["np_global"])
                torch.set_rng_state(cs["torch_cpu"])
                sys.stderr.write(">> resuming from %s at stage %d, iteration %d\n" % (checkpoint, start_stage, start_i))

        def snapshot(next_stage, next_i):                        # the loop's state at a step boundary (stage, i) -> next
            cpu = lambda t: None if t is None else t.detach().cpu()    # noqa: E731
            state = dict(
                images=[s.state() for s in st], adv_mask=cpu(adv_mask), adv_pattern=cpu(adv_pattern),
                mask_best=cpu(mask_best), pattern_best=cpu(pattern_best), have_stale=bool(have_stale),
                stale_gp=cpu(stale_gp) if have_stale else None, adv_x_prev=cpu(adv_x_prev),
                last_preds=None if last_preds is None else torch.from_numpy(np.ascontiguousarray(last_preds)),
                steps=int(steps), scans=[int(v) for v in scans], seeds=list(seeds) if on_device else None,
                rngs=[None if r is None or r is np.random else rng_state_out(r) for r in rngs],
                eot_rng=rng_state_out(eot_rng), np_global=rng_state_out(np.random), torch_cpu=torch.get_rng_state())
            return dict(version=CHECKPOINT_VERSION, fingerprint=fingerprint, stage=int(next_stage), i=int(next_i),
                        state=state)

        from concurrent.futures import ThreadPoolExecutor
        sampler = ThreadPoolExecutor(max_workers=1)
        prefetched = None

        for stage in range(start_stage, 2):
            first = start_i if stage == start_stage else 0       # > 0: resumed inside the stage, its start already ran
            if first == 0:
                print('============= Stage %d =============' % stage)
                for s in st:
                    s.reset()
                if stage == 0 and dir_0 and os.path.exists(os.path.join(dir_0, "adv_mask_%d.pt" % batch_id)):
                    mask_best = torch.load(os.path.join(dir_0, "adv_mask_%d.pt" % batch_id)).to(dev)
                    pattern_best = torch.load(os.path.join(dir_0, "adv_pattern_%d.pt" % batch_id)).to(dev)
                    continue
                if stage == 1:                                   # attack.py:143-165
                    adv_x, _, _ = eng.paste(x, mask_best, pattern_best, eps)
                    if any(not s.targeted for s in st):
                        p1 = eng.predict(adv_x)
                        for b, s in enumerate(st):
                            if not s.targeted:
                                s.targeted = True
                                s.y, sw = _pick_target(p1[b:b + 1], s.y)
                                s.crit_targeted = s.crit_targeted or sw
                    pattern_best = adv_x.clone()
                    torch.nn.Conv2d(1, 1, basic_unit, stride=basic_unit, bias=False)   # attack.py:365 RNG draw
                    adv_mask = self.patch_selection(mask_best, patch_budget, basic_unit, selection)
                    mask_best = adv_mask.clone()
                    adv_pattern = pattern_best.clone()
                adv_x_prev = None
            adv_x = None
            for i in range(first, max_iterations):
                if stage == 0 and i == 500:                      # attack.py:169-182
                    for b, s in enumerate(st):
                        if s.targeted or not s.active:
                            continue
                        s.targeted = True
                        y_new, sw = _pick_target(last_preds[b], s.y)
                        if y_new != s.y:
                            s.y = y_new
                            print(">> switch to targeted attack to category {:3d} at iteration: {:4d}".format(s.y, i))
                        s.crit_targeted = s.crit_targeted or sw
                        s.reset()
                        s.set_failed(scan(b, adv_x_prev))
                if stage == 0 and i == 499 and any(s.active and not s.targeted for s in st):
                    adv_x_prev, _, _ = eng.paste(x, adv_mask, adv_pattern, eps)   # the `adv_x` step 500 scans
                if i % 100 == 0:                                 # attack.py:187-190
                    adv_x, _, _ = eng.paste(x, adv_mask, adv_pattern, eps)
                    for b, s in enumerate(st):
                        if s.active:
                            s.set_failed(scan(b, adv_x))
                if prefetched is not None and prefetched[0] == (stage, i):
                    idx, idx2, nff, rects = prefetched[1].result()
                else:
                    idx, idx2, nff, rects = draw(i)
                prefetched = None
                # Draw step i+1's samples on a helper thread while the GPU runs step i -- only where the reference's RNG
                # consumption is provably unchanged: the draw depends on nothing this step can alter (i+1 < 1000: no
                # failed-set samples), the stage does run an iteration i+1, and no image can stop at step i (a stop needs
                # lr * 0.1 < 1e-3 together with a plateau, i.e. not_decay >= PATIENCE before the step).  Not before a
                # checkpoint either: the RNG states it saves must not hold step i+1's draw yet.
                ckpt_after = checkpoint is not None and (i + 1) % checkpoint_every == 0 and i + 1 < max_iterations
                if not on_device and not ckpt_after and _may_prefetch(st, i, max_iterations):
                    prefetched = ((stage, i + 1), sampler.submit(draw, i + 1))
                if dist and i % 100 == 0:
                    # every rank must have drawn the same indices (same RNG streams): a diverged rank would evaluate a
                    # slice of a different sample set and the gathered losses would be book-kept against the wrong masks
                    _assert_same_on_all_ranks(dist, idx, dev, "EOT sample indices at step %d" % i)
                structured_used = [s.structured for s in st]
                coeff_used = [s.coeff_group_lasso for s in st]
                xf = None
                if use_eot:
                    from . import eot as _eot
                    xf = _eot.sample(eot_rng, B, S, eot_affine, eot_colour)[:, rank * S_loc:(rank + 1) * S_loc]
                r = eng.attack_grad(x, adv_mask, adv_pattern, rects, [s.y for s in st],
                                    [s.crit_targeted for s in st], confidence, eps, stage, G, S_total=S, xforms=xf,
                                    basic_unit=basic_unit, S=S_loc)
                loss_adv, preds = r["loss_adv"], r["preds"]
                reduce_work = None
                if dist:                                         # one all-reduce of the patch gradient per step, under the bookkeeping
                    loss_adv, preds, reduce_work = exchange_shards(dist, G, loss_adv, preds, defer=True)
                last_preds = preds
                loss_target = r["group_lasso"] if stage == 0 else r["loss_struc"]
                counts = None
                if on_device:                                    # on the drawn indices, which never left the device
                    counts = eng.failed_update_drawn(B, S, [s.active for s in st], loss=loss_adv if dist else None)
                elif device_sets:                                # attack.py:259-267 as one kernel over the bitmaps; the host reads set sizes only
                    counts = eng.failed_update(idx, nff, [s.active for s in st], loss=loss_adv if dist else None)
                lr_used = np.zeros(B, np.float32)
                stopped_now = []
                for b, s in enumerate(st):
                    if not s.active:
                        continue
                    improved, stop = s.bookkeeping(stage, i, loss_adv[b], None if on_device else idx[b],
                                                   None if on_device else nff[b], loss_target[b],
                                                   n_failed=None if counts is None else counts[b])
                    if stop:
                        stopped_now.append(b)
                    if improved:                                 # best snapshot stays on the device
                        if stage == 0:
                            mask_best[b].copy_(adv_mask[b])
                        pattern_best[b].copy_(adv_pattern[b])
                    if stop:
                        print("early stop at iteration: {:4d}".format(i))
                        if np.isinf(s.loss_best):
                            mask_best[b].copy_(adv_mask[b])
                            pattern_best[b].copy_(adv_pattern[b])
                        s.active = False
                    else:
                        lr_used[b] = s.lr
                steps += 1
                if reduce_work is not None:                      # the sign step (and the stale-gradient capture) need the reduced G
                    reduce_work.wait()
                if stage == 0 and stopped_now:                   # capture the gradient the reference leaves in .grad
                    gp_full = torch.empty_like(x)
                    eng.attack_update(x, adv_mask, adv_pattern, G, np.zeros(B, np.float32), structured_used, coeff_used,
                                      density, stage, clip_min, clip_max, grad_pattern_out=gp_full)
                    for b in stopped_now:
                        stale_gp[b].copy_(gp_full[b])
                    have_stale = True
                if not any(s.active for s in st):
                    break
                if i % 20 == 0:                                  # attack.py:317-330
                    ys = np.asarray([s.y for s in st])[:, None]
                    acc = float((preds == ys).sum()) / (B * S) * 100
                    coef_st = np.asarray(structured_used, np.float32)
                    total = loss_adv.mean(1) + np.where(coef_st != 0, coef_st * r["loss_struc"], 0)
                    if stage == 0:
                        total = total + np.float32(density) * r["loss_density"] + \
                            np.asarray(coeff_used, np.float32) * r["group_lasso"]
                    msg = "iteration: {:4d}, accuracy: {:.2f}, loss: {:.2f}, adv: {:.2f}, l2 norm: {:.2f}, structural: {:.2f}".format(
                        i, acc, float(total.mean()), float(loss_adv.mean()),
                        float(np.minimum(r["l2"], eps).mean()), float(r["loss_struc"].mean()))
                    if stage == 0:
                        msg += ", group lasso: {:.2f}, density: {:.2f}".format(
                            float(r["group_lasso"].mean()), float(r["loss_density"].mean()))
                    print(msg)
                bias = stale_gp if (stage == 1 and i == 0 and have_stale) else None
                eng.attack_update(x, adv_mask, adv_pattern, G, lr_used, structured_used, coeff_used, density, stage,
                                  clip_min, clip_max, grad_pattern_bias=bias)   # attack.py:332-342
                if ckpt_after:
                    write_checkpoint(checkpoint, lambda: snapshot(stage, i + 1), dist)
            for b, s in enumerate(st):                           # attack.py:344-346
                if s.active and np.isinf(s.loss_best):
                    mask_best[b].copy_(adv_mask[b])
                    pattern_best[b].copy_(adv_pattern[b])
            if stage == 0:                                       # attack.py:348-359
                if dir_0 and rank == 0:
                    os.makedirs(dir_0, exist_ok=True)
                    torch.save(mask_best, os.path.join(dir_0, "adv_mask_%d.pt" % batch_id))
                    torch.save(pattern_best, os.path.join(dir_0, "adv_pattern_%d.pt" % batch_id))
                for b, s in enumerate(st):
                    if not s.targeted and last_preds is not None:
                        s.y, sw = _pick_target(last_preds[b], s.y)
                        s.crit_targeted = s.crit_targeted or sw
                if checkpoint is not None:                       # after the end-of-stage work, which must not rerun
                    write_checkpoint(checkpoint, lambda: snapshot(1, 0), dist)
        sampler.shutdown(wait=True)
        if checkpoint is not None:
            remove_checkpoint(checkpoint, dist)
        self.last_stats = dict(steps=steps, samples_per_step=B * S, final_labels=[s.y for s in st],
                               scans=scans[0], scan_forwards=scans[1])
        return mask_best, pattern_best

    # ------------------------------------------------------------------------------------
    def patch_selection(self, mask, patch_budget, basic_unit=7, selection='topk'):
        """attack.py:363-382: top-k basic_unit x basic_unit groups with positive importance -> binary mask.
        Window sums on the device (native kernel); the k-of-(H/basic_unit)^2 selection on the host."""
        if selection != 'topk':
            raise NotImplementedError("selection=%r" % (selection,))
        from .runtime import shared_engine
        B, _, H, W = mask.shape
        eng = shared_engine(W, B)
        imp = eng.window_sum(mask.contiguous().float(), basic_unit)                   # [B, (H/u)*(W/u)]
        num_group = int(np.floor((H * W * patch_budget) / (basic_unit ** 2)))
        sel = np.zeros_like(imp)
        for b in range(B):
            order = np.argsort(-imp[b], kind="stable")[:num_group]
            sel[b, order[imp[b, order] > 0]] = 1
        sel = torch.from_numpy(sel.reshape(B, 1, H // basic_unit, W // basic_unit)).to(mask.device)
        return sel.repeat_interleave(basic_unit, dim=2).repeat_interleave(basic_unit, dim=3)

    def collect_failure(self, adv_x, y, mask_set_universe, targeted, model, batch_size=128, transforms=None):
        """attack.py:384-406 with the reference's signature: `mask_set_universe` may be the bool
        tensor of the reference or an int16 rectangle table [n,2,4]."""
        bank = None
        if not isinstance(mask_set_universe, np.ndarray):
            # the reference's bool universe [n,1,H,W] (True = keep): masks that are "all but <= 2 rectangles" take the
            # rectangle path of the native K1 kernel; any other universe is packed into a mask bank (dp_predict_bank)
            if transforms is not None:
                raise NotImplementedError("collect_failure(transforms=...) is an unused hook of the reference (attack.py:395-396)")
            try:
                mask_set_universe = _masks.from_bool(mask_set_universe)
            except NotImplementedError:
                bank = _masks.pack_bank(mask_set_universe, device=adv_x.device)
        net = unwrap_native(model)
        eng = net.engine(adv_x.shape[-1], max_images=adv_x.shape[0])
        B = adv_x.shape[0]
        if bank is None:
            n = mask_set_universe.shape[0]
            rects = _masks.gather(mask_set_universe, np.arange(n))
            preds = eng.predict(adv_x.contiguous().float(), n, np.broadcast_to(rects, (B,) + rects.shape))
        else:
            n = bank.shape[0]
            preds = eng.predict(adv_x.contiguous().float(), n, bank=bank, idx=np.tile(np.arange(n), B))
        yv = np.asarray(y.tolist() if torch.is_tensor(y) else y).reshape(B, -1)[:, :1]
        f = preds.reshape(B, n) == yv
        if targeted:
            f = ~f
        failed = np.nonzero(f.any(0))[0].tolist()
        print(">> %d failures collected!" % len(failed))
        return failed
