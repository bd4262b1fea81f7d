"""Oracle restatement of the classifier the reference attacks.

The reference builds ``timm.create_model('resnetv2_50x1_bit_distilled')``
(reference utils.py:51-58) and wraps it in ``NormModel`` with
mean=std=0.5 (reference utils.py:66-78).  timm 0.6.7 is a third-party
dependency that is not vendored in the reference and not installed here, so the
architecture is restated from its published definition (timm 0.6.7
``models/resnetv2.py``: ResNetV2 with PreActBottleneck blocks, StdConv2d
weight-standardised convolutions eps=1e-8, GroupNorm(32)+ReLU, 'fixed' stem) and
cross-checked against ``transformers.models.bit`` in the tests.

Pure torch-CPU functional code over a flat ``{timm_key: tensor}`` dict.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import math

import torch
import torch.nn.functional as F

DEPTHS = (3, 4, 6, 3)
WIDTHS = (256, 512, 1024, 2048)
STEM_CH = 64
GN_GROUPS = 32
GN_EPS = 1e-5
WS_EPS = 1e-8


def param_shapes(num_classes=1000):
    """timm-named parameter shapes of resnetv2_50x1_bit (state_dict order)."""
    shapes = {"stem.conv.weight": (STEM_CH, 3, 7, 7)}
    cin = STEM_CH
    for s, (depth, cout) in enumerate(zip(DEPTHS, WIDTHS)):
        mid = cout // 4
        for b in range(depth):
            p = "stages.%d.blocks.%d." % (s, b)
            if b == 0:
                shapes[p + "downsample.conv.weight"] = (cout, cin, 1, 1)
            shapes[p + "norm1.weight"] = (cin,)
            shapes[p + "norm1.bias"] = (cin,)
            shapes[p + "conv1.weight"] = (mid, cin, 1, 1)
            shapes[p + "norm2.weight"] = (mid,)
            shapes[p + "norm2.bias"] = (mid,)
            shapes[p + "conv2.weight"] = (mid, mid, 3, 3)
            shapes[p + "norm3.weight"] = (mid,)
            shapes[p + "norm3.bias"] = (mid,)
            shapes[p + "conv3.weight"] = (cout, mid, 1, 1)
            cin = cout
    shapes["norm.weight"] = (cin,)
    shapes["norm.bias"] = (cin,)
    shapes["head.fc.weight"] = (num_classes, cin, 1, 1)
    shapes["head.fc.bias"] = (num_classes,)
    return shapes


def random_init(seed=0, num_classes=1000, affine_jitter=0.0):
    """Deterministic random-init weights (no checkpoint is available offline).

    Conv weights: N(0, 2/fan_out) (every conv, *including* conv3 -- timm's
    zero_init_last would make every residual branch dead at init, which is
    useless for a synthetic benchmark).  GroupNorm: weight 1, bias 0 (plus an
    optional jitter so tests exercise the affine path).  fc: N(0, 0.01), bias 0.
    The same recipe is implemented (independently) in
    dorpatch_b200/resnetv2.py; tests check both produce identical tensors.
    """
    g = torch.Generator().manual_seed(seed)
    params = {}
    for name, shp in param_shapes(num_classes).items():
        if len(shp) == 4 and name != "head.fc.weight":
            fan_out = shp[0] * shp[2] * shp[3]
            params[name] = torch.randn(shp, generator=g) * math.sqrt(2.0 / fan_out)
        elif name == "head.fc.weight":
            params[name] = torch.randn(shp, generator=g) * 0.01
        elif name == "head.fc.bias":
            params[name] = torch.zeros(shp)
        elif name.endswith("weight"):  # GroupNorm gamma
            params[name] = torch.ones(shp)
            if affine_jitter:
                params[name] += affine_jitter * torch.randn(shp, generator=g)
        else:  # GroupNorm beta
            params[name] = torch.zeros(shp)
            if affine_jitter:
                params[name] += affine_jitter * torch.randn(shp, generator=g)
    return params


def standardize(w, eps=WS_EPS):
    """timm StdConv2d: per-output-channel (w-mean)/sqrt(biased_var+eps)."""
    flat = w.reshape(w.shape[0], -1)
    mean = flat.mean(1, keepdim=True)
    var = flat.var(1, unbiased=False, keepdim=True)
    return ((flat - mean) / torch.sqrt(var + eps)).reshape(w.shape)


def _gn_relu(x, w, b):
    return F.relu(F.group_norm(x, GN_GROUPS, w, b, GN_EPS))


def forward_features(params, z, taps=None):
    """z: normalised input [N,3,H,W] -> pre-head feature map [N,2048,h,w]."""
    ws = standardize
    x = F.conv2d(z, ws(params["stem.conv.weight"]), stride=2, padding=3)
    if taps is not None:
        taps["stem"] = x
    x = F.pad(x, (1, 1, 1, 1), value=0.0)          # ConstantPad2d(1, 0.)
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=0)
    if taps is not None:
        taps["pool"] = x
    for s, depth in enumerate(DEPTHS):
        for b in range(depth):
            p = "stages.%d.blocks.%d." % (s, b)
            stride = 2 if (b == 0 and s > 0) else 1
            xp = _gn_relu(x, params[p + "norm1.weight"], params[p + "norm1.bias"])
            if b == 0:
                shortcut = F.conv2d(xp, ws(params[p + "downsample.conv.weight"]), stride=stride)
            else:
                shortcut = x
            h = F.conv2d(xp, ws(params[p + "conv1.weight"]))
            h = _gn_relu(h, params[p + "norm2.weight"], params[p + "norm2.bias"])
            h = F.conv2d(h, ws(params[p + "conv2.weight"]), stride=stride, padding=1)
            h = _gn_relu(h, params[p + "norm3.weight"], params[p + "norm3.bias"])
            h = F.conv2d(h, ws(params[p + "conv3.weight"]))
            x = h + shortcut
            if taps is not None:
                taps["s%db%d" % (s, b)] = x
    return x


def forward_normalized(params, z, taps=None):
    """Logits for an already-normalised input (what timm's model sees)."""
    x = forward_features(params, z, taps)
    x = _gn_relu(x, params["norm.weight"], params["norm.bias"])
    x = x.mean((2, 3), keepdim=True)
    x = F.conv2d(x, params["head.fc.weight"], params["head.fc.bias"])
    return x.flatten(1)


def forward(params, x01, taps=None):
    """NormModel.forward (reference utils.py:77-78): (x-0.5)/0.5 -> net."""
    return forward_normalized(params, (x01 - 0.5) / 0.5, taps)


class OracleNet(torch.nn.Module):
    """nn.Module view so the oracle (and the shimmed reference) can call
    ``model(x)`` with x in [0,1].  ``requires_grad`` on the weights mirrors the
    reference, which never freezes them (main.py:51-55; SURVEY quirk Q7)."""

    def __init__(self, params, weights_require_grad=True):
        super().__init__()
        self.keys = list(params.keys())
        self.plist = torch.nn.ParameterList(
            [torch.nn.Parameter(params[k].clone(), requires_grad=weights_require_grad) for k in self.keys])

    def pdict(self):
        return {k: p for k, p in zip(self.keys, self.plist)}

    def forward(self, x01):
        return forward(self.pdict(), x01)
