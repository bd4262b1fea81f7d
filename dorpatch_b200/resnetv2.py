"""ResNetV2-50x1-BiT parameter container whose forward runs on the native engine.

The reference obtains this classifier from timm (``timm.create_model(
'resnetv2_50x1_bit_distilled')``, reference utils.py:51-58).  timm is not vendored
there; this module keeps timm's parameter names (``stem.conv.weight``,
``stages.S.blocks.B.{downsample.conv,norm1,conv1,norm2,conv2,norm3,conv3}``, ``norm``,
``head.fc``) so PatchCleanser checkpoints load with ``load_state_dict``, and executes on
libdorpatch.so.  There is deliberately no PyTorch-eager forward: without a CUDA device (or
without the built library) ``forward`` raises.
"""
import math
import os

import torch
from torch import nn

# Product default = the reference's own GPU arithmetic (fp32 storage, TF32 tensor-core convolutions: PyTorch's
# cudnn.allow_tf32 default).  bf16 is opt-in (DORPATCH_PRECISION=bf16 / --precision bf16); its end-metric parity
# evidence is tests/test_gpu_attack_success.py.
DEFAULT_PRECISION = "tf32"

DEPTHS = (3, 4, 6, 3)
WIDTHS = (256, 512, 1024, 2048)
STEM_CH = 64


def param_shapes(num_classes=1000):
    """{timm name: shape} of every parameter, in state-dict order (no tensors allocated)."""
    sh = {"stem.conv.weight": (STEM_CH, 3, 7, 7)}
    cin = STEM_CH
    for s, (depth, cout) in enumerate(zip(DEPTHS, WIDTHS)):
        for b in range(depth):
            c0, mid, p = (cin if b == 0 else cout), cout // 4, "stages.%d.blocks.%d." % (s, b)
            if b == 0:
                sh[p + "downsample.conv.weight"] = (cout, c0, 1, 1)
            sh[p + "norm1.weight"] = sh[p + "norm1.bias"] = (c0,)
            sh[p + "conv1.weight"] = (mid, c0, 1, 1)
            sh[p + "norm2.weight"] = sh[p + "norm2.bias"] = (mid,)
            sh[p + "conv2.weight"] = (mid, mid, 3, 3)
            sh[p + "norm3.weight"] = sh[p + "norm3.bias"] = (mid,)
            sh[p + "conv3.weight"] = (cout, mid, 1, 1)
        cin = cout
    sh["norm.weight"] = sh["norm.bias"] = (cin,)
    sh["head.fc.weight"] = (num_classes, cin, 1, 1)
    sh["head.fc.bias"] = (num_classes,)
    return sh


class _Conv(nn.Module):          # holds `.weight` (OIHW), standardised by the engine at load time
    def __init__(self, cin, cout, k):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k))


class _Norm(nn.Module):          # GroupNorm(32) affine parameters
    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))


class _Downsample(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = _Conv(cin, cout, 1)


class _Block(nn.Module):
    def __init__(self, cin, cout, first):
        super().__init__()
        mid = cout // 4
        if first:
            self.downsample = _Downsample(cin, cout)
        self.norm1, self.conv1 = _Norm(cin), _Conv(cin, mid, 1)
        self.norm2, self.conv2 = _Norm(mid), _Conv(mid, mid, 3)
        self.norm3, self.conv3 = _Norm(mid), _Conv(mid, cout, 1)


class _Stage(nn.Module):
    def __init__(self, cin, cout, depth):
        super().__init__()
        self.blocks = nn.ModuleList([_Block(cin if b == 0 else cout, cout, b == 0) for b in range(depth)])


class _Stem(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = _Conv(3, STEM_CH, 7)


class _Head(nn.Module):
    def __init__(self, cin, num_classes):
        super().__init__()
        self.fc = nn.Conv2d(cin, num_classes, 1, bias=True)


class ResNetV2(nn.Module):
    """timm-compatible ``resnetv2_50x1_bit`` container; forward = native engine."""

    def __init__(self, num_classes=1000, seed=0):
        super().__init__()
        self.num_classes = num_classes
        self.stem = _Stem()
        cin, stages = STEM_CH, []
        for depth, cout in zip(DEPTHS, WIDTHS):
            stages.append(_Stage(cin, cout, depth))
            cin = cout
        self.stages = nn.ModuleList(stages)
        self.norm = _Norm(cin)
        self.head = _Head(cin, num_classes)
        self._engines = {}
        self._version = 0
        self._param_grads = False
        self.init_weights(seed)

    def reset_classifier(self, num_classes):
        """timm API used by the reference (utils.py:58)."""
        if num_classes != self.num_classes:
            self.num_classes = num_classes
            self.head = _Head(WIDTHS[-1], num_classes)
            nn.init.normal_(self.head.fc.weight, 0.0, 0.01)
            nn.init.zeros_(self.head.fc.bias)
            self.invalidate()

    def init_weights(self, seed=0):
        """Deterministic random init (no checkpoint is reachable offline): conv N(0, 2/fan_out)
        for every conv -- timm's zero_init_last would leave every residual branch dead --
        GroupNorm weight 1 / bias 0, fc N(0, 0.01) / bias 0."""
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p in self.state_dict().items():
                if p.dim() == 4 and name != "head.fc.weight":
                    fan_out = p.shape[0] * p.shape[2] * p.shape[3]
                    p.copy_(torch.randn(p.shape, generator=g) * math.sqrt(2.0 / fan_out))
                elif name == "head.fc.weight":
                    p.copy_(torch.randn(p.shape, generator=g) * 0.01)
                elif name.endswith("bias"):
                    p.zero_()
                else:
                    p.fill_(1.0)
        self.invalidate()

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.invalidate()
        return r

    def invalidate(self):
        """Weights changed: engines must re-standardise them."""
        self._version += 1

    def param_grads_(self, on=True):
        """Weight gradients through the engine for ``model(x)`` / ``NormModel`` / ``DataParallel`` (fine-tuning): the
        parameters that require grad get ``.grad`` (``ops.eot_logits(..., param_grads=True)``), and the logits are
        differentiable even when x does not require grad.  Off by default; returns self."""
        self._param_grads = bool(on)
        return self

    def _param_state(self):
        return {k: (p._version, p.data_ptr()) for k, p in self.named_parameters()}

    def _refresh(self, eng):
        """Reload the parameters changed in place since `eng` was loaded (an optimizer step, ``p.copy_``): their
        ``_version`` counters / storage moved.  Through the device, into the same engine."""
        cur = self._param_state()
        held = getattr(eng, "_weights_state", None)
        if held is None:
            eng._weights_state = cur
            return eng
        changed = [k for k, v in cur.items() if held.get(k) != v]
        if changed:
            params = dict(self.named_parameters())
            eng.load_state_dict_dev({k: params[k] for k in changed})
            eng._weights_state = cur
        return eng

    # ------------------------------------------------------------------------------
    def engine(self, img, max_images=1, precision=None, chunk=None):
        """The native engine for this model at image size `img` (created on first use)."""
        from .engine import Engine
        forced = getattr(self, "_adopted", None)
        if forced is not None and forced.handle and forced.img == int(img) and forced.max_images >= max_images:
            return self._refresh(forced)
        precision = precision or os.environ.get("DORPATCH_PRECISION", DEFAULT_PRECISION)
        chunk = int(chunk or os.environ.get("DORPATCH_CHUNK", "128"))
        key = (int(img), precision, chunk, torch.cuda.current_device() if torch.cuda.is_available() else -1)
        ent = self._engines.get(key)
        if ent is not None and (ent[1] != self._version or ent[0].max_images < max_images):
            ent[0].close()
            ent = None
        if ent is None:
            # DORPATCH_AUTOTUNE=0: library algorithms by heuristic instead of timing trials, the same in every process
            eng = Engine(img=img, n_classes=self.num_classes, precision=precision, chunk=chunk,
                         max_images=max(int(max_images), 1),
                         autotune=os.environ.get("DORPATCH_AUTOTUNE", "1") != "0")
            eng.load_state_dict({k: v for k, v in self.state_dict().items()})
            eng._weights_state = self._param_state()
            from . import runtime
            runtime.register(eng)          # weight-free helpers (utils.clip, patch_selection) reuse it
            ent = (eng, self._version)
            self._engines[key] = ent
        return self._refresh(ent[0])

    def adopt_engine(self, eng):
        """Use an engine the caller already built (and loaded with THESE weights) instead of creating one."""
        self._adopted = eng
        eng._weights_state = self._param_state()

    def forward(self, z):
        """Logits of an already-normalised batch [N,3,H,W] (what timm's module computes).  Differentiable with
        respect to z when z requires grad (``ops.eot_logits`` on z * 0.5 + 0.5, so the engine sees z up to one
        rounding); the parameters get no gradient unless ``param_grads_(True)``."""
        if not z.is_cuda:
            raise RuntimeError("dorpatch_b200.ResNetV2 runs on the native CUDA engine only (no CPU fallback)")
        if torch.is_grad_enabled() and (z.requires_grad or self._param_grads):
            from .ops import eot_logits
            return eot_logits(self, z.float() * 0.5 + 0.5, param_grads=self._param_grads)
        eng = self.engine(z.shape[-1])
        z = z.contiguous().float()
        outs = [eng.net_forward_backward(z[i:i + eng.chunk]) for i in range(0, z.shape[0], eng.chunk)]
        return torch.cat(outs, 0)

    def forward_unit(self, x01):
        """Logits for images in [0,1] (NormModel with mean=std=0.5 fused into K1)."""
        eng = self.engine(x01.shape[-1], max_images=1)
        _, logits = eng.predict(x01.contiguous().float(), 1, None, return_logits=True)
        return torch.from_numpy(logits).to(x01.device)
