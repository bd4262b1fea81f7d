"""Differentiable native classifier: ``eot_logits`` puts the engine's forward and backward-to-input behind
``torch.autograd``, so any loss written in PyTorch can drive a patch attack (cross-entropy, a top-k margin, an
adaptive attack on the PatchCleanser decision, ...), not only the CW loss that ``dp_attack_grad`` has built in.

    logits = eot_logits(model, adv_x, rects, S)          # [B*S, K] = model(occlude(adv_x_b, rects[b, s]))
    F.cross_entropy(logits, y.repeat_interleave(S)).backward()
    adv_x.grad                                           # [B, 3, H, W]

The forward is ``dp_eot_forward`` (K1 + the classifier, the logits bit for bit those of ``dp_predict``); the
backward is ``dp_eot_backward`` (classifier backward + K1^T on the current stream).  What is differentiated:

- the image only.  The classifier's parameters get no ``.grad``: the engine has no weight-gradient pass.
- once.  ``create_graph=True`` (double backward) raises.
- the engine's last forward.  A backward after another forward on the same engine (``eot_logits`` again,
  ``dp_predict`` / PatchCleanser, ``generate``) raises instead of returning a gradient of the wrong activations.
  ``retain_graph=True`` and repeated backwards of the same forward are fine.
"""
import torch

from .utils import unwrap_native


class _EotLogits(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, eng, S, rects):
        logits = eng.eot_forward(img, S, rects)
        ctx.eng, ctx.token = eng, eng.eot_forwards
        ctx.save_for_backward(img)                    # autograd then refuses a backward after an in-place change
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        if torch.is_grad_enabled():
            raise RuntimeError("eot_logits: double backward (create_graph=True) is not supported; the engine computes "
                               "first-order input gradients only")
        img, = ctx.saved_tensors
        eng = ctx.eng
        if eng.eot_forwards != ctx.token:
            raise RuntimeError("eot_logits: the engine ran another eot_forward after this one; its activations are "
                               "gone, so this graph can no longer be differentiated (run the forward again)")
        return eng.eot_backward(dlogits.contiguous().float()), None, None, None


def eot_logits(model, img, rects=None, S=1):
    """Differentiable ``model(occlude(img))``: [B*S, K] logits, sample b*S+s occluding image b with rects[b, s].

    model: ``ResNetV2``, ``NormModel(ResNetV2)`` or ``DataParallel`` of either (the native engine; anything else
    raises TypeError).  img: [B, 3, H, W] CUDA tensor in [0, 1]; NormModel's (x - 0.5) / 0.5 is fused into K1.
    rects: [B, S, 4, 4] int16 rectangle tables (``masks.gather``), or None for plain classification (S = 1).
    Differentiable with respect to ``img`` only (see the module docstring)."""
    net = unwrap_native(model)
    if not (isinstance(img, torch.Tensor) and img.is_cuda):
        raise RuntimeError("eot_logits runs on the native CUDA engine only (no CPU fallback)")
    S = int(S)
    if rects is None and S != 1:
        raise ValueError("eot_logits: S=%d needs rectangle tables (rects=None is plain classification, S=1)" % S)
    if img.dim() != 4 or img.shape[1] != 3:
        raise ValueError("eot_logits: img must be [B, 3, H, W], got %s" % (tuple(img.shape),))
    eng = net.engine(img.shape[-1], max_images=img.shape[0])
    return _EotLogits.apply(img.contiguous().float(), eng, S, rects)
