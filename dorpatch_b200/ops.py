"""Differentiable native classifier: ``eot_logits`` puts the engine's forward and backward-to-input behind
``torch.autograd``, so any loss written in PyTorch can drive a patch attack (cross-entropy, a top-k margin, an
adaptive attack on the PatchCleanser decision, ...), not only the CW loss that ``dp_attack_grad`` has built in.

    logits = eot_logits(model, adv_x, rects, S)          # [B*S, K] = model(occlude(adv_x_b, rects[b, s]))
    F.cross_entropy(logits, y.repeat_interleave(S)).backward()
    adv_x.grad                                           # [B, 3, H, W]

The forward is ``dp_eot_forward`` (K1 + the classifier, the logits bit for bit those of ``dp_predict``); the
backward is ``dp_eot_backward`` (classifier backward + K1^T on the current stream).  What is differentiated:

- the image.  The classifier's parameters get no ``.grad`` by default.  With ``param_grads=True`` (or
  ``ResNetV2.param_grads_(True)`` for ``model(x)``) the parameters that require grad are inputs too, and the backward
  is ``dp_eot_backward_params``: the engine's weight-gradient pass, run only for those parameters (fine-tuning under
  cutout / adversarial fine-tuning).  ``.grad`` then accumulates exactly as for an ``nn.Module``; after
  ``optimizer.step()`` the engine reloads the changed weights on its next use.  With ``xforms`` (affine / colour EOT,
  ``dp_eot_forward_xform``) the transform parameters get no gradient.
- once.  ``create_graph=True`` (double backward) raises.
- the engine's last forward.  A backward after another forward on the same engine (``eot_logits`` again,
  ``dp_predict`` / PatchCleanser, ``generate``) raises instead of returning a gradient of the wrong activations.
  ``retain_graph=True`` and repeated backwards of the same forward are fine.
"""
import numpy as np
import torch

from .utils import unwrap_native


class _EotLogits(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, eng, S, rects, xforms, bank, idx, names, *params):
        logits = eng.eot_forward(img, S, rects, xforms, bank=bank, idx=idx)
        ctx.eng, ctx.token, ctx.names = eng, eng.eot_forwards, names
        ctx.banked = bank is not None
        # autograd then refuses a backward after an in-place change of the image or the bank
        ctx.save_for_backward(img, *((bank,) if ctx.banked else ()), *params)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        if torch.is_grad_enabled():
            raise RuntimeError("eot_logits: double backward (create_graph=True) is not supported; the engine computes "
                               "first-order input gradients only")
        saved = ctx.saved_tensors
        params = saved[2:] if ctx.banked else saved[1:]
        none = (None,) * 7                              # eng, S, rects, xforms, bank, idx, names
        eng = ctx.eng
        if eng.eot_forwards != ctx.token:
            raise RuntimeError("eot_logits: the engine ran another eot_forward after this one; its activations are "
                               "gone, so this graph can no longer be differentiated (run the forward again)")
        d = dlogits.contiguous().float()
        if ctx.names is None:
            return (eng.eot_backward(d),) + none
        live = [i for i in range(len(params)) if ctx.needs_input_grad[8 + i]]
        grads = [torch.empty(params[i].shape, dtype=torch.float32, device=d.device) for i in live]
        g_img = eng.eot_backward_params(d, [ctx.names[i] for i in live], grads, grad_img=ctx.needs_input_grad[0])
        out = [None] * len(params)
        for i, g in zip(live, grads):
            out[i] = g if g.device == params[i].device else g.to(params[i].device)
        return (g_img,) + none + tuple(out)


def _check_xforms(xforms, img, S):
    """[B, S, 8] float32 host array of the transforms, or TypeError / ValueError."""
    if isinstance(xforms, torch.Tensor):
        if not xforms.dtype.is_floating_point:
            raise TypeError("eot_logits: xforms must be a float tensor, got %s" % xforms.dtype)
        xforms = xforms.detach().cpu().numpy()
    xforms = np.asarray(xforms)
    if xforms.dtype.kind != "f":
        raise TypeError("eot_logits: xforms must be a float array, got %s" % xforms.dtype)
    B = img.shape[0] if isinstance(img, torch.Tensor) and img.dim() >= 1 else None
    if xforms.ndim != 3 or xforms.shape[1:] != (S, 8) or (B is not None and xforms.shape[0] != B):
        raise ValueError("eot_logits: xforms must be [B, S, 8] with B = %s, S = %d, got %s" % (B, S, xforms.shape))
    return np.ascontiguousarray(xforms, dtype=np.float32)


def _check_bank(bank, idx, img, S):
    """idx of a mask bank as a [B*S, 2] int32 host array, or TypeError / ValueError."""
    if not (isinstance(bank, torch.Tensor) and bank.dtype == torch.int32 and bank.dim() == 3):
        raise TypeError("eot_logits: bank must be the int32 tensor [M, H, ceil(W/32)] of masks.pack_bank")
    if idx is None:
        raise ValueError("eot_logits: a bank needs idx, [B, S] or [B, S, 2] mask indices")
    if isinstance(idx, torch.Tensor):
        idx = idx.detach().cpu().numpy()
    idx = np.asarray(idx)
    if idx.dtype.kind not in "iu":
        raise TypeError("eot_logits: idx must be an integer array, got %s" % idx.dtype)
    B = img.shape[0] if isinstance(img, torch.Tensor) and img.dim() >= 1 else None
    if idx.ndim == 2:
        idx = np.stack([idx, np.full(idx.shape, -1, idx.dtype)], axis=-1)
    if idx.ndim != 3 or idx.shape[1:] != (S, 2) or (B is not None and idx.shape[0] != B):
        raise ValueError("eot_logits: idx must be [B, S] or [B, S, 2] with B = %s, S = %d, got %s" % (B, S, idx.shape))
    M = int(bank.shape[0])
    if idx.size and (idx.min() < -1 or idx.max() >= M):
        raise ValueError("eot_logits: idx holds mask indices outside [-1, %d)" % M)
    return np.ascontiguousarray(idx, dtype=np.int32)


def eot_logits(model, img, rects=None, S=1, xforms=None, param_grads=False, bank=None, idx=None):
    """Differentiable ``model(occlude(img))``: [B*S, K] logits, sample b*S+s occluding image b with rects[b, s].

    model: ``ResNetV2``, ``NormModel(ResNetV2)`` or ``DataParallel`` of either (the native engine; anything else
    raises TypeError).  img: [B, 3, H, W] CUDA tensor in [0, 1]; NormModel's (x - 0.5) / 0.5 is fused into K1.
    rects: [B, S, 4, 4] int16 rectangle tables (``masks.gather``), or None: plain classification (S = 1), or no
    occlusion when xforms are given.
    xforms: [B, S, 8] float tensor or array of affine / colour transforms, e.g. ``eot.sample(rng, B, S, affine,
    colour)``: sample b*S+s is ``clamp(c * (grid_sample(img_b, affine_grid(theta)) - 0.5) + 0.5 + br, 0, 1)``
    (bilinear, border padding, align_corners=False; theta = xforms[b, s, :6] as 2 x 3, c, br = xforms[b, s, 6:]),
    then occluded -- what ``generate(eot_affine=..., eot_colour=...)`` optimises against.  None: no transform.
    Differentiable with respect to ``img``; the transform parameters get no gradient (see the module docstring).
    With xforms the input gradient is summed with fp32 atomics, so its last bits can differ from run to run.
    param_grads: also differentiate the classifier's fp32 parameters that require grad (frozen ones get None and
    cost nothing); the logits are then differentiable even when img does not require grad.
    bank / idx: occlude with arbitrary masks instead of rectangles: bank = ``masks.pack_bank(keep)`` (bool keep-masks
    [M, 1, H, W], True = keep), idx [B, S] or [B, S, 2] int mask indices (sample b*S+s is occluded where mask
    idx[b, s, 0] or idx[b, s, 1] is, -1 = none).  Not with rects or xforms.  The bank is saved for the backward like
    img: changing it in place before the backward raises."""
    net = unwrap_native(model)
    if bank is not None:
        if rects is not None:
            raise ValueError("eot_logits: give rects or a bank, not both")
        if xforms is not None:
            raise ValueError("eot_logits: a bank cannot be combined with xforms (the warped path reads rectangles)")
        idx = _check_bank(bank, idx, img, int(S))
    elif idx is not None:
        raise ValueError("eot_logits: idx without a bank")
    if not isinstance(param_grads, bool):
        raise TypeError("eot_logits: param_grads must be True or False, got %r" % (param_grads,))
    names, params = None, ()
    if param_grads:
        named = [(k, p) for k, p in net.named_parameters() if p.requires_grad]
        for k, p in named:
            if p.dtype != torch.float32:
                raise TypeError("eot_logits: param_grads needs fp32 parameters; %s is %s" % (k, p.dtype))
        names, params = tuple(k for k, _ in named), tuple(p for _, p in named)
    if xforms is not None:
        xforms = _check_xforms(xforms, img, int(S))
    if not (isinstance(img, torch.Tensor) and img.is_cuda):
        raise RuntimeError("eot_logits runs on the native CUDA engine only (no CPU fallback)")
    S = int(S)
    if rects is None and S != 1 and xforms is None and bank is None:
        raise ValueError("eot_logits: S=%d needs rectangle tables or xforms (rects=None without xforms is plain "
                         "classification, S=1)" % S)
    if img.dim() != 4 or img.shape[1] != 3:
        raise ValueError("eot_logits: img must be [B, 3, H, W], got %s" % (tuple(img.shape),))
    eng = net.engine(img.shape[-1], max_images=img.shape[0])
    return _EotLogits.apply(img.contiguous().float(), eng, S, rects, xforms, bank, idx, names, *params)
