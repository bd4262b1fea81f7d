"""Python handle on one native DorPatch engine (one per GPU).

Thin: converts torch CUDA tensors / numpy host arrays to the raw pointers of the C ABI
(include/dorpatch.h) and raises RuntimeError on any native error.  PyTorch is plumbing here
(device memory, the current stream); all compute is in libdorpatch.so.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

PRECISIONS = {"fp32": 0, "tf32": 1, "bf16": 2}


def _dev_ptr(t, dtype=torch.float32):
    if t is None:
        return None
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise TypeError("expected a CUDA tensor")
    if t.dtype != dtype:
        raise TypeError("expected dtype %s, got %s" % (dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


def _host(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    return a, C.c_void_p(a.ctypes.data)


class Engine:
    """ResNetV2-50x1-BiT attack engine on one CUDA device."""

    def __init__(self, img=224, n_classes=1000, precision="bf16", chunk=64, max_images=1, device=None,
                 autotune=True):
        if not torch.cuda.is_available():
            raise RuntimeError("dorpatch_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.img, self.n_classes, self.precision = int(img), int(n_classes), precision
        self.chunk, self.max_images = int(chunk), int(max_images)
        cfg = _lib.DpConfig(self.device, self.img, self.n_classes, PRECISIONS[precision], self.chunk,
                            self.max_images, 1 if autotune else 0, 0)
        h = C.c_void_p()
        _lib.check(self.lib.dp_engine_create(C.byref(cfg), C.byref(h)))
        self.handle = h
        cp, eb = C.c_int32(), C.c_int32()
        _lib.check(self.lib.dp_input_layout(self.handle, C.byref(cp), C.byref(eb)))
        self.c_pad, self.elem_bytes = cp.value, eb.value
        self.failed_masks = 4096                 # capacity of the failed-mask sets until failed_reset
        self.eot_forwards = 0                    # eot_forward calls so far (ops.eot_logits pairs a backward with its forward)
        self._eot_shape = None

    def close(self):
        if getattr(self, "handle", None):
            self.lib.dp_engine_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def device_bytes(self):
        return int(self.lib.dp_engine_device_bytes(self.handle))

    @property
    def launch_count(self):
        return int(self.lib.dp_engine_launch_count(self.handle))

    @property
    def graph_replays(self):
        return int(self.lib.dp_engine_graph_replays(self.handle))

    @property
    def graph_status(self):
        return self.lib.dp_engine_graph_status(self.handle).decode("utf-8", "replace")

    def profile(self, enable=True, reset=False):
        """Per-category CUDA-event profiler of the engine's launches (adds sync overhead)."""
        _lib.check(self.lib.dp_engine_profile(self.handle, 2 if (enable and reset) else (1 if enable else 0)))

    def profile_read(self):
        """-> {category: dict(ms, bytes, flops, count)} accumulated since the last reset."""
        n, stride = 64, 32
        names = C.create_string_buffer(n * stride)
        ms, by, fl = (C.c_double * n)(), (C.c_double * n)(), (C.c_double * n)()
        cnt = (C.c_int64 * n)()
        got = C.c_int32()
        _lib.check(self.lib.dp_engine_profile_read(self.handle, n, C.cast(names, C.c_void_p), stride, C.cast(ms, C.c_void_p),
                                                   C.cast(by, C.c_void_p), C.cast(fl, C.c_void_p), C.cast(cnt, C.c_void_p),
                                                   C.byref(got)))
        out = {}
        for i in range(got.value):
            nm = names.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode()
            out[nm] = dict(ms=ms[i], bytes=by[i], flops=fl[i], count=int(cnt[i]))
        return out

    def load_state_dict(self, state_dict):
        """timm-named fp32 tensors of resnetv2_50x1_bit (utils.py:57-62 of the reference)."""
        names, arrs = [], []
        for k, v in state_dict.items():
            names.append(k.encode())
            arrs.append(np.ascontiguousarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v,
                                             dtype=np.float32))
        n = len(names)
        c_names = (C.c_char_p * n)(*names)
        c_ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        c_num = (C.c_int64 * n)(*[a.size for a in arrs])
        _lib.check(self.lib.dp_engine_load_weights(self.handle, n, c_names, c_ptrs, c_num))

    def load_state_dict_dev(self, state_dict, names=None):
        """Reload timm-named tensors (any subset) from fp32 CUDA tensors on this engine's device, without a host copy
        and without rebuilding the engine (dp_engine_load_weights_dev).  Invalidates the last eot_forward."""
        keys = list(state_dict.keys()) if names is None else list(names)
        tens = []
        for k in keys:
            v = state_dict[k].detach()
            if not v.is_cuda or v.device.index != self.device:
                v = v.to("cuda:%d" % self.device)
            tens.append(v.float().contiguous())
        n = len(keys)
        c_names = (C.c_char_p * n)(*[k.encode() for k in keys])
        c_ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in tens])
        c_num = (C.c_int64 * n)(*[t.numel() for t in tens])
        _lib.check(self.lib.dp_engine_load_weights_dev(self.handle, n, c_names, c_ptrs, c_num, self._stream()))
        self.eot_forwards += 1                   # the engine's last forward is gone

    # ------------------------------------------------------------------------------
    def paste(self, x, mask, pattern, eps, out=None):
        """adv_x = x + clip(mask, pattern, x, eps); returns (adv_x, l2[B], scale[B])."""
        B = x.shape[0]
        out = torch.empty_like(x) if out is None else out
        l2 = np.empty(B, np.float32)
        sc = np.empty(B, np.float32)
        _lib.check(self.lib.dp_paste(self.handle, _dev_ptr(x), _dev_ptr(mask), _dev_ptr(pattern), B, float(eps),
                                     _dev_ptr(out), C.c_void_p(l2.ctypes.data), C.c_void_p(sc.ctypes.data),
                                     self._stream()))
        return out, l2, sc

    def window_sum(self, t, k, square=False):
        B = t.shape[0]
        g = self.img // k
        out = np.empty((B, g * g), np.float32)
        _lib.check(self.lib.dp_window_sum(self.handle, _dev_ptr(t), B, int(k), 1 if square else 0,
                                          C.c_void_p(out.ctypes.data), self._stream()))
        return out

    def expand(self, img, S, rects=None):
        """K1 alone (tests / profiling): returns the network-input tensor
        [B*S, H, W, c_pad] in the engine's activation dtype."""
        B = img.shape[0]
        N = B * S
        dt = torch.bfloat16 if self.elem_bytes == 2 else torch.float32
        out = torch.empty((N, self.img, self.img, self.c_pad), dtype=dt, device=img.device)
        rp = None
        if rects is not None:
            rects, rp = _host(np.asarray(rects).reshape(N, 4, 4), np.int16)
        _lib.check(self.lib.dp_expand(self.handle, _dev_ptr(img), B, S, rp, C.c_void_p(out.data_ptr()),
                                      self._stream()))
        return out

    def predict(self, img, S=1, rects=None, return_logits=False):
        """argmax of model(occlude(img)) for S occlusions per image; img [B,3,H,W] in [0,1]."""
        B = img.shape[0]
        N = B * S
        preds = np.empty(N, np.int32)
        logits = np.empty((N, self.n_classes), np.float32) if return_logits else None
        rp = None
        if rects is not None:
            rects, rp = _host(np.asarray(rects).reshape(N, 4, 4), np.int16)
        _lib.check(self.lib.dp_predict(self.handle, _dev_ptr(img), B, S, rp, C.c_void_p(preds.ctypes.data),
                                       C.c_void_p(logits.ctypes.data) if return_logits else None, self._stream()))
        return (preds, logits) if return_logits else preds

    # ------------------------------------------------------------------------------
    def eot_forward(self, img, S=1, rects=None, xforms=None):
        """model(occlude(img)) as [B*S, K] logits on the device (dp_predict's values), keeping what eot_backward needs.
        img [B,3,H,W] fp32 in [0,1]; rects [B,S,4,4] int16 or None (then S must be 1 unless xforms are given).
        xforms: [B,S,8] affine / colour transforms (eot.sample's layout) applied before the occlusion, or None."""
        B = img.shape[0]
        N = B * int(S)
        logits = torch.empty((N, self.n_classes), dtype=torch.float32, device=img.device)
        rp = None
        if rects is not None:
            rects, rp = _host(np.asarray(rects).reshape(N, 4, 4), np.int16)
        if xforms is None:
            _lib.check(self.lib.dp_eot_forward(self.handle, _dev_ptr(img), B, int(S), rp, _dev_ptr(logits),
                                               self._stream()))
        else:
            if isinstance(xforms, torch.Tensor):
                xforms = xforms.detach().cpu().numpy()
            xf, xp = _host(np.asarray(xforms).reshape(N, 8), np.float32)
            _lib.check(self.lib.dp_eot_forward_xform(self.handle, _dev_ptr(img), B, int(S), rp, xp, _dev_ptr(logits),
                                                     self._stream()))
        self.eot_forwards += 1
        self._eot_shape = tuple(img.shape)
        return logits

    def eot_backward(self, dlogits, out=None):
        """d<dlogits, logits>/d img of the last eot_forward, [B,3,H,W] (weight gradients: eot_backward_params)."""
        out = torch.empty(self._eot_shape, dtype=torch.float32, device=dlogits.device) if out is None else out
        _lib.check(self.lib.dp_eot_backward(self.handle, _dev_ptr(dlogits), _dev_ptr(out), self._stream()))
        return out

    def eot_backward_params(self, dlogits, names, grads, grad_img=True, accumulate=False):
        """eot_backward plus parameter gradients (dp_eot_backward_params): grads[i] (fp32 CUDA, contiguous, the shape of
        timm tensor names[i]) receives d<dlogits, logits>/d tensor (written, or added with accumulate=True).
        grad_img: True -> return the image gradient [B,3,H,W]; a tensor -> written there; False / None -> skipped."""
        out = None
        if grad_img is True:
            out = torch.empty(self._eot_shape, dtype=torch.float32, device=dlogits.device)
        elif isinstance(grad_img, torch.Tensor):
            out = grad_img
        n = len(names)
        if len(grads) != n:
            raise ValueError("eot_backward_params: %d names but %d gradient buffers" % (n, len(grads)))
        from .resnetv2 import param_shapes
        shapes = param_shapes(self.n_classes)
        for k, g in zip(names, grads):          # the C ABI carries no sizes: a short buffer would be written past its end
            if k not in shapes:
                raise ValueError("eot_backward_params: unknown parameter name %r" % (k,))
            want = int(np.prod(shapes[k]))
            if not (isinstance(g, torch.Tensor) and g.is_cuda and g.dtype == torch.float32 and g.is_contiguous()):
                raise TypeError("eot_backward_params: the gradient buffer of %s must be a contiguous fp32 CUDA tensor" % k)
            if g.numel() != want:
                raise ValueError("eot_backward_params: the gradient buffer of %s has %d elements, %s has %d"
                                 % (k, g.numel(), k, want))
        c_names = (C.c_char_p * n)(*[k.encode() for k in names])
        c_ptrs = (C.c_void_p * n)(*[_dev_ptr(g).value for g in grads])
        _lib.check(self.lib.dp_eot_backward_params(self.handle, _dev_ptr(dlogits), _dev_ptr(out), n, c_names, c_ptrs,
                                                   1 if accumulate else 0, self._stream()))
        return out

    def attack_grad(self, x, mask, pattern, rects, y, crit_targeted, confidence, eps, stage, grad_adv,
                    S_total=None, host=False, xforms=None, basic_unit=7):
        """attack.py:184-247.  rects [B,S,4,4] int16; y [B]; crit_targeted [B] bool; basic_unit: side of the
        group-lasso groups (must divide H), which the following attack_update also uses.
        Fills grad_adv [B,3,H,W] and returns a dict of host numpy results."""
        B = x.shape[0]
        rects = np.ascontiguousarray(rects, dtype=np.int16)
        S = rects.size // (B * 16)
        N = B * S
        yh, yp = _host(y, np.int64)
        th, tp = _host(crit_targeted, np.uint8)
        res = dict(loss_adv=np.empty((B, S), np.float32), preds=np.empty((B, S), np.int32),
                   loss_struc=np.empty(B, np.float32), loss_density=np.zeros(B, np.float32),
                   group_lasso=np.zeros(B, np.float32), l2=np.empty(B, np.float32))
        a = _lib.DpAttackArgs()
        a.B, a.S, a.S_total, a.stage = B, S, int(S_total or S), int(stage)
        a.basic_unit = int(basic_unit)
        if host:
            self._keep = [np.ascontiguousarray(t, np.float32) for t in (x, mask, pattern)]
            a.x, a.mask, a.pattern = [t.ctypes.data for t in self._keep]
            a.grad_adv = None
        else:
            a.x, a.mask, a.pattern = _dev_ptr(x), _dev_ptr(mask), _dev_ptr(pattern)
            a.grad_adv = _dev_ptr(grad_adv)
        a.rects_host = rects.ctypes.data
        a.y_host, a.targeted_host = yp, tp
        a.confidence, a.eps = float(confidence), float(eps)
        a.loss_adv_host = res["loss_adv"].ctypes.data
        a.preds_host = res["preds"].ctypes.data
        a.loss_struc_host = res["loss_struc"].ctypes.data
        a.loss_density_host = res["loss_density"].ctypes.data
        a.group_lasso_host = res["group_lasso"].ctypes.data
        a.l2_host = res["l2"].ctypes.data
        xf = None
        if xforms is not None:        # optional affine / colour EOT: [B,S,8] float32
            xf = np.ascontiguousarray(xforms, dtype=np.float32).reshape(N, 8)
            a.xform_host = xf.ctypes.data
        self._live = (rects, yh, th, res, xf)
        if host:
            return a, res
        _lib.check(self.lib.dp_attack_grad(self.handle, C.byref(a), self._stream()))
        return res

    def _update_args(self, x, mask, pattern, grad_adv, lr, structured, coeff_gl, density, stage, clip_min,
                     clip_max, grad_pattern_out, grad_mask_out, host=False, grad_pattern_bias=None):
        B = x.shape[0]
        u = _lib.DpUpdateArgs()
        u.B, u.stage = B, int(stage)
        lrh, lrp = _host(lr, np.float32)
        sth, stp = _host(structured, np.float32)
        cgh, cgp = _host(coeff_gl if coeff_gl is not None else np.zeros(B), np.float32)
        if host:
            u.x, u.mask, u.pattern = x.ctypes.data, mask.ctypes.data, pattern.ctypes.data
            u.grad_adv = None
        else:
            u.x, u.mask, u.pattern, u.grad_adv = _dev_ptr(x), _dev_ptr(mask), _dev_ptr(pattern), _dev_ptr(grad_adv)
            u.grad_pattern_out = _dev_ptr(grad_pattern_out)
            u.grad_mask_out = _dev_ptr(grad_mask_out)
            u.grad_pattern_bias = _dev_ptr(grad_pattern_bias)
        u.lr_host, u.structured_host, u.coeff_gl_host = lrp, stp, cgp
        u.density, u.clip_min, u.clip_max = float(density), float(clip_min), float(clip_max)
        self._live_u = (lrh, sth, cgh)
        return u

    def attack_update(self, x, mask, pattern, grad_adv, lr, structured, coeff_gl, density, stage,
                      clip_min=0.0, clip_max=1.0, grad_pattern_out=None, grad_mask_out=None, grad_pattern_bias=None):
        """attack.py:332-342 (in place on mask / pattern)."""
        u = self._update_args(x, mask, pattern, grad_adv, lr, structured, coeff_gl, density, stage, clip_min,
                              clip_max, grad_pattern_out, grad_mask_out, grad_pattern_bias=grad_pattern_bias)
        _lib.check(self.lib.dp_attack_update(self.handle, C.byref(u), self._stream()))

    def attack_step_host(self, x, mask, pattern, rects, y, crit_targeted, confidence, eps, stage, lr, structured,
                         coeff_gl, density, S_total=None, clip_min=0.0, clip_max=1.0):
        """One whole step through HOST numpy buffers (mask / pattern updated in place)."""
        a, res = self.attack_grad(x, mask, pattern, rects, y, crit_targeted, confidence, eps, stage, None,
                                  S_total=S_total, host=True)
        xs, ms, ps = self._keep
        u = self._update_args(xs, ms, ps, None, lr, structured, coeff_gl, density, stage, clip_min,
                              clip_max, None, None, host=True)
        _lib.check(self.lib.dp_attack_step_host(self.handle, C.byref(a), C.byref(u), self._stream()))
        return res

    # ------------------------------------------------------------------------------
    # failed-mask sets on the device (attack.py:96,187-190,259-267)
    def failed_reset(self, n_mask):
        """Size every image's failed set for a universe of n_mask masks and clear it (default capacity: 4096)."""
        _lib.check(self.lib.dp_failed_set_reset(self.handle, int(n_mask), self._stream()))
        self.failed_masks = int(n_mask)

    def failed_write(self, b, indices):
        a, p = _host(np.asarray(indices, dtype=np.int32).reshape(-1), np.int32)
        _lib.check(self.lib.dp_failed_set_write(self.handle, int(b), p, int(a.size), self._stream()))

    def failed_update(self, idx, nff, active, loss=None, thresh=0.1):
        """One step of attack.py:259-267 for every image; returns the set sizes [B]."""
        idx, ip = _host(idx, np.int32)
        B, S = idx.shape
        nf, np_ = _host(nff, np.int32)
        ac, ap = _host(active, np.uint8)
        lp = None
        if loss is not None:
            loss, lp = _host(loss, np.float32)
        cnt = np.empty(B, np.int32)
        _lib.check(self.lib.dp_failed_set_update(self.handle, B, S, ip, np_, ap, lp, float(thresh), C.c_void_p(cnt.ctypes.data), self._stream()))
        return cnt

    def failed_read(self, b):
        out = np.empty(self.failed_masks, np.int32)
        n = C.c_int32()
        _lib.check(self.lib.dp_failed_set_read(self.handle, int(b), C.c_void_p(out.ctypes.data), out.size,
                                               C.cast(C.byref(n), C.c_void_p), self._stream()))
        return out[:n.value].tolist()

    # ------------------------------------------------------------------------------
    def net_forward_backward(self, z, dlogits=None):
        """Classifier on a normalised NCHW batch (test hook): logits [N,K] (+ dz)."""
        N = z.shape[0]
        logits = torch.empty((N, self.n_classes), dtype=torch.float32, device=z.device)
        dz = torch.empty_like(z) if dlogits is not None else None
        _lib.check(self.lib.dp_net_forward_backward(self.handle, _dev_ptr(z), N, _dev_ptr(logits),
                                                    _dev_ptr(dlogits), _dev_ptr(dz), self._stream()))
        return (logits, dz) if dlogits is not None else logits
