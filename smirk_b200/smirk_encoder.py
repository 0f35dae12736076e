"""``SmirkEncoder`` — drop-in for the reference ``src/smirk_encoder.py`` (eval BN).

Same class names, constructor arguments, sub-module / parameter names (``state_dict`` keys follow the
timm ``features_only`` MobileNetV3 layout the reference checkpoints use) and output dicts.  The
``nn.Conv2d`` / ``nn.BatchNorm2d`` objects below are parameter containers only — they are never
called; the forward pass runs in ``csrc/encoder.cu`` through ``smk_encoder_forward``.

With grad mode on and an image that requires grad, a frozen (``requires_grad_(False)``) encoder whose BatchNorms are in
eval mode passes the gradient to its input, as the reference trainer's cycle loss (its encoder frozen by
``utils.freeze_module``) and analysis-by-synthesis fitting need: the forward then keeps its activations
(``smk_encoder_forward_saved``) and the backward runs ``smk_encoder_backward``.

Train mode (``.train()``, what the reference trainer runs) is opt-in: per module with ``allow_train_mode_(True)``, or
process-wide with ``set_train_mode_default(True)`` (``python -m smirk_b200.dropin --train``).  Then the BatchNorms
normalise with batch statistics and update their running statistics (``smk_encoder_forward_train``), and every parameter
that requires grad gets its gradient (``smk_encoder_backward_train``).  Batch statistics couple the images of a batch.
Without the opt-in a train-mode encoder raises; eval-mode weight gradients are not implemented.

Live weights (``live_weights_(True)``, off by default) run the eval path on a handle whose folded BatchNorms and packed
operands are refreshed on the device from the module's own tensors at every call (``smk_encoder_refresh``), instead of
a handle packed on the host whenever a parameter or buffer changes: no host round trip, no allocation, and a CUDA graph of
the call reads the weights and running statistics of replay time.  It suits a frozen encoder whose weights another path
keeps training (the second path of the trainer's step); fixed inference weights keep the host-packed handle, which a
captured graph (``SmirkPipeline.capture``) holds at the weights of capture time.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib

BN_EPS = 1e-3          # timm tf_* models (BN_EPS_TF_DEFAULT)
# The process-wide train-mode opt-in, one flag shared with SmirkGenerator (it lives in _lib).
set_train_mode_default = _lib.set_train_mode_default
train_mode_default = _lib.train_mode_default

# (kind, stride, expansion, out_channels) per block, grouped per stage — timm 0.9.16
# tf_mobilenetv3_{large,small}_minimal_100 with features_only=True (stops after the `cn` stage).
ARCH = {
    "tf_mobilenetv3_large_minimal_100": [
        [("ds", 1, 1.0, 16)],
        [("ir", 2, 4.0, 24), ("ir", 1, 3.0, 24)],
        [("ir", 2, 3.0, 40), ("ir", 1, 3.0, 40), ("ir", 1, 3.0, 40)],
        [("ir", 2, 6.0, 80), ("ir", 1, 2.5, 80), ("ir", 1, 2.3, 80), ("ir", 1, 2.3, 80)],
        [("ir", 1, 6.0, 112), ("ir", 1, 6.0, 112)],
        [("ir", 2, 6.0, 160), ("ir", 1, 6.0, 160), ("ir", 1, 6.0, 160)],
        [("cn", 1, 1.0, 960)],
    ],
    "tf_mobilenetv3_small_minimal_100": [
        [("ds", 2, 1.0, 16)],
        [("ir", 2, 4.5, 24), ("ir", 1, 3.67, 24)],
        [("ir", 2, 4.0, 40), ("ir", 1, 6.0, 40), ("ir", 1, 6.0, 40)],
        [("ir", 1, 3.0, 48), ("ir", 1, 3.0, 48)],
        [("ir", 2, 6.0, 96), ("ir", 1, 6.0, 96), ("ir", 1, 6.0, 96)],
        [("cn", 1, 1.0, 576)],
    ],
}


def _make_divisible(v, divisor=8, round_limit=0.9):
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    if new_v < round_limit * v:
        new_v += divisor
    return new_v


def _conv(cin, cout, k, stride=1, groups=1):
    return nn.Conv2d(cin, cout, k, stride=stride, groups=groups, bias=False)


def _bn(c):
    return nn.BatchNorm2d(c, eps=BN_EPS)


class _Block(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("smirk_b200: backbone blocks are parameter containers; call SmirkEncoder.forward")


class _DS(_Block):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv_dw, self.bn1 = _conv(cin, cin, 3, stride, cin), _bn(cin)
        self.conv_pw, self.bn2 = _conv(cin, cout, 1), _bn(cout)


class _IR(_Block):
    def __init__(self, cin, cout, stride, exp):
        super().__init__()
        mid = _make_divisible(cin * exp)
        self.conv_pw, self.bn1 = _conv(cin, mid, 1), _bn(mid)
        self.conv_dw, self.bn2 = _conv(mid, mid, 3, stride, mid), _bn(mid)
        self.conv_pwl, self.bn3 = _conv(mid, cout, 1), _bn(cout)


class _CN(_Block):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv, self.bn1 = _conv(cin, cout, 1), _bn(cout)


class _Backbone(_Block):
    """Parameter tree of a timm MobileNetV3Features model (conv_stem, bn1, blocks.<stage>.<i>...)."""

    def __init__(self, name):
        super().__init__()
        self.conv_stem, self.bn1 = _conv(3, 16, 3, 2), _bn(16)
        stages, cin = [], 16
        for stage in ARCH[name]:
            blocks = []
            for kind, s, e, c in stage:
                blocks.append(_DS(cin, c, s) if kind == "ds" else _IR(cin, c, s, e) if kind == "ir" else _CN(cin, c))
                cin = c
            stages.append(nn.Sequential(*blocks))
        self.blocks = nn.Sequential(*stages)
        self.feature_dim = cin

    def tensor_list(self):
        """fp32 tensors in state_dict order without num_batches_tracked (the C ABI's contract)."""
        return [v for k, v in self.state_dict().items() if not k.endswith("num_batches_tracked")]


def create_backbone(backbone_name, pretrained=True):
    """Signature of smirk_encoder.py:7-12.  ``pretrained`` is accepted and ignored: there is no network
    access here and the reference always overwrites the weights from its checkpoint (demo.py:55-58)."""
    bb = _Backbone(backbone_name)
    return bb, bb.feature_dim


class _NativeEncoder(_lib.NativeModule, nn.Module):
    """Shared machinery of SmirkEncoder and its three sub-encoders: a native handle over the backbones returned by
    ``_parts()`` (slot 0 = pose / small, 1 = shape / large, 2 = expression / large; None = not part of this module),
    re-packed whenever a parameter / buffer is modified or moved, and the raw forward through the C ABI.

    ``precision``: 0 fp32 CUDA cores | 1 TF32 wgmma 1x1 convs | 2 = 1 + fused expand/depthwise blocks |
    3 = 2 with error-compensated 3xTF32 arithmetic (fp32-equivalent; the parity path)."""

    def _init_native(self, n_exp=50, n_shape=300):
        self.n_exp, self.n_shape = n_exp, n_shape
        self.precision = 0

    def _parts(self):
        raise NotImplementedError

    def _native_extras(self):
        return (self.precision,)

    def _native_create(self, device):
        keep = []
        d = _lib.SmkEncoderDesc()
        for i, part in enumerate(self._parts()):
            if part is None:
                d.n_tensors[i] = 0
                continue
            enc, head = part
            ts = enc.encoder.tensor_list()
            arr = (_lib.c_f32p * len(ts))()
            for j, t in enumerate(ts):
                a, p = _lib.f32(t)
                keep.append(a)
                arr[j] = p
            keep.append(arr)
            d.tensors[i] = C.cast(arr, C.POINTER(_lib.c_f32p))
            d.n_tensors[i] = len(ts)
            a, p = _lib.f32(head.weight); keep.append(a); d.head_w[i] = p
            a, p = _lib.f32(head.bias); keep.append(a); d.head_b[i] = p
        d.n_shape, d.n_exp, d.precision = self.n_shape, self.n_exp, int(self.precision)
        return _lib.create("encoder", d, device)

    def allow_train_mode_(self, on=True):
        """Opt this module and its sub-encoders in to (or out of) train mode; returns the module."""
        for m in self.modules():
            if isinstance(m, _NativeEncoder):
                m._allow_train = bool(on)
        return self

    def live_weights_(self, on=True):
        """Run the eval path of this module and its sub-encoders on weights refreshed on the device at every call (see the
        module docstring); returns the module."""
        for m in self.modules():
            if isinstance(m, _NativeEncoder):
                m._live = bool(on)
        return self

    def _live_tensors(self):
        """The tensors a refresh reads, flat: per backbone its ``encoder`` tensors in state_dict order without
        num_batches_tracked (conv weight, BN weight, bias, running_mean, running_var per conv), then the head's weight and
        bias."""
        out = []
        for part in self._parts():
            if part is not None:
                enc, head = part
                out += [v for k, v in enc.encoder.state_dict(keep_vars=True).items() if not k.endswith("num_batches_tracked")]
                out += [head.weight, head.bias]
        return out

    def _live_handle(self, dev):
        present = tuple(p is not None for p in self._parts())
        mask = sum(1 << i for i, p in enumerate(present) if p)
        return _lib.live_handle(self, "encoder", dev, (present, self.n_shape, self.n_exp, int(self.precision)),
                                (mask, self.n_shape, self.n_exp, int(self.precision)))

    def _refresh(self, h, dev, tensors):
        """smk_encoder_refresh of live handle h from ``_live_tensors()`` (or the tensors an autograd context saved)."""
        a, keep = _lib.SmkEncoderTrainArgs(), []
        it = iter(tensors)
        ptr = lambda t: C.cast(t.data_ptr(), _lib.c_f32p)
        for i, part in enumerate(self._parts()):
            if part is None:
                continue
            bns = [m for m in part[0].encoder.modules() if isinstance(m, nn.BatchNorm2d)]
            eps = {m.eps for m in bns}
            if len(eps) != 1:
                raise RuntimeError("smirk_b200.%s: live weights need one eps for all BatchNorms of a backbone, got %s"
                                   % (type(self).__name__, sorted(eps)))
            ts = [next(it) for _ in range(5 * len(bns) + 2)]
            for t in ts:
                _check_param(t, dev)
            arr = (_lib.c_f32p * (len(ts) - 2))(*[ptr(t) for t in ts[:-2]])
            keep.append(arr)
            a.tensors[i] = C.cast(arr, C.POINTER(_lib.c_f32p))
            a.n_tensors[i] = len(ts) - 2
            a.head_w[i], a.head_b[i] = ptr(ts[-2]), ptr(ts[-1])
            a.eps[i] = eps.pop()
        _lib.refresh("encoder", h, dev, a)

    def _eval_handle(self, dev):
        """-> (handle, tensors): the host-packed eval handle and None, or with live weights the live handle, refreshed
        from the tensors returned."""
        if not self.__dict__.get("_live"):
            return self._native_handle(dev), None
        h, tensors = self._live_handle(dev), self._live_tensors()
        self._refresh(h, dev, tensors)
        return h, tensors

    def _train_allowed(self):
        on = self.__dict__.get("_allow_train")
        return _lib.train_mode_default() if on is None else on

    def _check(self, img):
        """Device, shape and mode checks of every call -> True for a train-mode call.  The mode is that of the BatchNorms
        the call runs, as in the reference (whose parent module owns none): a parent in train mode over frozen, eval-mode
        sub-encoders runs the eval path."""
        _lib.require_cuda(img, "img")
        name = type(self).__name__
        modes = []
        for part in self._parts():            # checked on every call: .train() after the first forward must not silently run eval BN
            if part is not None:
                modes.append({m.training for m in part[0].encoder.modules() if isinstance(m, nn.BatchNorm2d)})
        train = any(True in m for m in modes)
        if train and not self._train_allowed():
            raise RuntimeError("smirk_b200.%s: train-mode BatchNorm runs only with the opt-in: call .allow_train_mode_(True) on "
                               "the encoder or run under `python -m smirk_b200.dropin --train`" % name)
        if train and any(m != {True} for m in modes):
            raise RuntimeError("smirk_b200.%s: one call runs backbones whose BatchNorms mix train and eval mode; call the "
                               "sub-encoders (pose_encoder, shape_encoder, expression_encoder) separately" % name)
        if img.dim() != 4 or tuple(img.shape[1:]) != (3, 224, 224):
            raise RuntimeError("smirk_b200.%s: expected img [B,3,224,224], got %s" % (name, tuple(img.shape)))
        if train:
            for part in self._parts():
                if part is not None:
                    _bn_settings(part[0].encoder, name)
        return train

    def _outputs(self, B, dev):
        widths = (6, self.n_shape, self.n_exp + 5)
        return [torch.empty(B, w, dtype=torch.float32, device=dev) if part is not None else None
                for w, part in zip(widths, self._parts())]

    def _run(self, img):
        """img [B,3,224,224] -> (pose_cam [B,6] | None, shape [B,n_shape] | None, expr [B,n_exp+5] | None)."""
        if self._check(img):
            return self._run_train(img)
        if torch.is_grad_enabled() and img.requires_grad:
            parts = [p for p in self._parts() if p is not None]
            if any(t.requires_grad for enc, head in parts for t in list(enc.encoder.parameters()) + list(head.parameters())):
                raise RuntimeError("smirk_b200.%s: weight gradients are not implemented; to pass a gradient to the input, "
                                   "freeze the encoder with .requires_grad_(False)" % type(self).__name__)
            raw = _EncoderFunction.apply(img, self)
            it = iter(raw)
            return [next(it) if p is not None else None for p in self._parts()]
        with torch.no_grad():
            dev = img.device
            h = self._eval_handle(dev)[0]
            x = _lib.dev_f32(img, "img")
            B = x.shape[0]
            outs = self._outputs(B, dev)
            ws = self._native_workspace("forward", _lib.call("smk_encoder_workspace_bytes", dev, h, B), dev)
            _lib.call("smk_encoder_forward", dev, h, x, B, *outs, ws, ws.numel())
            return outs

    def _forward_saved(self, img):
        """-> (handle, outputs, saved) of ``_forward_saved_live``."""
        return self._forward_saved_live(img)[:3]

    def _forward_saved_live(self, img):
        """-> (handle, [raw outputs | None], saved, live tensors | None): the grad-mode forward, its activations in a buffer
        of their own."""
        dev = img.device
        h, tensors = self._eval_handle(dev)
        x = _lib.dev_f32(img, "img")
        B = x.shape[0]
        outs = self._outputs(B, dev)
        saved = _lib.saved_buffer("encoder", h, B, dev)
        ws = self._native_workspace("forward", _lib.call("smk_encoder_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_encoder_forward_saved", dev, h, x, B, *outs, saved, saved.numel() * 4, ws, ws.numel())
        return h, outs, saved, tensors

    @torch.no_grad()
    def saved_activations(self, img):
        """The tensors the backward of ``self(img)`` uses, {name: tensor}, names being the reference's module paths: the
        output of every ReLU as a [B,C,H,W] view of the NHWC buffer (``shape_encoder.encoder.bn1`` for the stem,
        ``….blocks.<stage>.<i>.bn1`` / ``.bn2`` ...) and each head's pre-clamp output [B,n_out]
        (``expression_encoder.expression_layers.0`` ...).  The forward is deterministic and batch-independent, so these
        are the tensors an autograd context of the same input holds."""
        if self._check(img):                 # train mode: on copies of the running statistics, which stay untouched
            h, _, saved = self._forward_train(img, self._train_params(), True, copy_stats=True)
        else:
            h, _, saved = self._forward_saved(img)
        return _lib.saved_views("encoder", h, saved, img.shape[0])

    # ---- train mode ---------------------------------------------------------------------------------------------------
    def _train_params(self):
        """The parameters of the backbones this module runs, flat: per backbone its ``encoder`` parameters (conv weight,
        BN weight, bias per conv, in state_dict order), then the head's weight and bias."""
        out = []
        for part in self._parts():
            if part is not None:
                out += list(part[0].encoder.parameters()) + [part[1].weight, part[1].bias]
        return out

    def _train_handle(self, dev):
        st = self._native
        present = tuple(p is not None for p in self._parts())
        key = (str(dev), present, self.n_shape, self.n_exp, int(self.precision))
        if st.train_handle is None or st.train_key != key:
            st.train_handle = None
            h = C.c_void_p()
            _lib.call("smk_encoder_train_create", dev, sum(1 << i for i, p in enumerate(present) if p), self.n_shape, self.n_exp,
                      int(self.precision), C.byref(h))
            st.train_handle, st.train_key = _lib.NativeHandle(h, "smk_encoder_destroy"), key
        return st.train_handle

    def _train_args(self, dev, params, copy_stats=False):
        """-> (SmkEncoderTrainArgs, keep-alive list, [(running_mean, running_var, num_batches_tracked)] per BN).  params:
        ``_train_params()`` (or the tensors an autograd context saved).  copy_stats: point at copies of the running
        statistics (a forward that must leave the module untouched)."""
        a, keep, stats = _lib.SmkEncoderTrainArgs(), [], []
        it = iter(params)
        ptr = lambda t: C.cast(t.data_ptr(), _lib.c_f32p)
        for i, part in enumerate(self._parts()):
            if part is None:
                continue
            enc, head = part
            bns = [m for m in enc.encoder.modules() if isinstance(m, nn.BatchNorm2d)]
            momentum, eps = _bn_settings(enc.encoder, type(self).__name__)
            ts, nbt = [], []
            for bn in bns:
                w, g, b = next(it), next(it), next(it)
                rm, rv, n = bn.running_mean, bn.running_var, bn.num_batches_tracked
                if copy_stats:
                    rm, rv, n = rm.clone(), rv.clone(), n.clone()
                for t in (w, g, b, rm, rv):
                    _check_param(t, dev)
                if n.device != dev or n.dtype != torch.int64:
                    raise RuntimeError("smirk_b200: num_batches_tracked must be an int64 tensor on %s" % dev)
                ts += [w, g, b, rm, rv]
                nbt.append(n)
                stats.append((rm, rv, n))
            hw, hb = next(it), next(it)
            _check_param(hw, dev); _check_param(hb, dev)
            arr = (_lib.c_f32p * len(ts))(*[ptr(t) for t in ts])
            narr = (C.POINTER(C.c_int64) * len(nbt))(*[C.cast(t.data_ptr(), C.POINTER(C.c_int64)) for t in nbt])
            keep += [arr, narr, ts, nbt]
            a.tensors[i] = C.cast(arr, C.POINTER(_lib.c_f32p))
            a.n_tensors[i] = len(ts)
            a.num_batches_tracked[i] = C.cast(narr, C.POINTER(C.POINTER(C.c_int64)))
            a.head_w[i], a.head_b[i] = ptr(hw), ptr(hb)
            a.momentum[i], a.eps[i] = -1.0 if momentum is None else momentum, eps
        return a, keep, stats

    def _forward_train(self, img, params, with_saved, copy_stats=False):
        """-> (handle, [raw outputs | None], saved | None): one train-mode forward, which updates the running statistics
        (of copies, with copy_stats)."""
        dev = img.device
        h = self._train_handle(dev)
        x = _lib.dev_f32(img, "img")
        B = x.shape[0]
        outs = self._outputs(B, dev)
        args, keep, stats = self._train_args(dev, params, copy_stats)
        nbytes = _lib.call("smk_encoder_train_workspace_bytes", dev, h, B)
        saved = _lib.saved_buffer("encoder", h, B, dev) if with_saved else None
        if saved is None:
            nbytes += _lib.call("smk_encoder_saved_bytes", dev, h, B)
        ws = self._native_workspace("train", nbytes, dev)
        _lib.call("smk_encoder_forward_train", dev, h, C.byref(args), x, B, *outs, saved,
                  0 if saved is None else saved.numel() * 4, ws, ws.numel())
        if not copy_stats:                  # the eval handle repacks, and copies see the new statistics
            for t in (t for s in stats for t in s):
                torch.autograd.graph.increment_version(t)
        return h, outs, saved

    def _run_train(self, img):
        params = self._train_params()
        if torch.is_grad_enabled() and (img.requires_grad or any(p.requires_grad for p in params)):
            raw = _EncoderTrainFunction.apply(img, self, *params)
            it = iter(raw)
            return [next(it) if p is not None else None for p in self._parts()]
        with torch.no_grad():
            return self._forward_train(img, params, False)[1]


def _bn_settings(backbone, name):
    """-> (momentum, eps) shared by every BatchNorm of a backbone (the kernels take one pair per backbone)."""
    bns = [m for m in backbone.modules() if isinstance(m, nn.BatchNorm2d)]
    settings = {(m.momentum, m.eps) for m in bns}
    if len(settings) != 1:
        raise RuntimeError("smirk_b200.%s: train mode needs one momentum and one eps for all BatchNorms of a backbone, got %s"
                           % (name, sorted(settings, key=str)))
    momentum, eps = settings.pop()
    if not all(m.affine and m.track_running_stats for m in bns):
        raise RuntimeError("smirk_b200.%s: train mode needs affine BatchNorms that track running statistics" % name)
    if (momentum is not None and not 0.0 <= momentum <= 1.0) or not eps > 0:
        raise RuntimeError("smirk_b200.%s: train mode takes momentum in [0, 1] or None and eps > 0, got momentum %r, eps %r"
                           % (name, momentum, eps))
    return momentum, eps


def _check_param(t, dev):
    if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
        raise RuntimeError("smirk_b200: train mode needs contiguous float32 parameters and buffers on %s" % dev)


class _EncoderFunction(torch.autograd.Function):
    """Frozen encoder: the raw outputs (pose_cam, shape, expr: those the module holds) of img, and the gradient with
    respect to img only.  An output that receives no gradient arrives as None and its backbone's backward launches
    nothing.  The activations are saved per call, so several forwards may share one backward.  With live weights the
    tensors the refresh read are saved too (autograd raises if one is modified in place before the backward), and the
    backward refreshes the handle from them again when another call has refreshed it since."""

    @staticmethod
    def forward(ctx, img, module):
        h, outs, saved, tensors = module._forward_saved_live(img)
        ctx.set_materialize_grads(False)
        ctx.handle, ctx.module, ctx.dtype, ctx.B = h, module, img.dtype, img.shape[0]
        ctx.present = [o is not None for o in outs]
        ctx.live = tensors is not None
        ctx.generation = h.generation if ctx.live else None
        ctx.save_for_backward(saved, *(tensors or ()))
        return tuple(o for o in outs if o is not None)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        saved, *tensors = ctx.saved_tensors
        m, dev, B = ctx.module, saved.device, ctx.B
        if ctx.live and ctx.handle.generation != ctx.generation:
            m._refresh(ctx.handle, dev, tensors)
            ctx.generation = ctx.handle.generation
        it = iter(grads)
        g = [next(it) if p else None for p in ctx.present]
        g = [None if t is None else _lib.dev_f32(t, "grad") for t in g]
        g_img = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev)
        ws = m._native_workspace("backward", _lib.call("smk_encoder_backward_workspace_bytes", dev, ctx.handle, B), dev)
        _lib.call("smk_encoder_backward", dev, ctx.handle, B, saved, saved.numel() * 4, *g, g_img, ws, ws.numel())
        return g_img.to(ctx.dtype), None


class _EncoderTrainFunction(torch.autograd.Function):
    """Train-mode encoder: the raw outputs (those the module holds) of img, and the gradients of img and of every
    parameter in ``_train_params()`` order.  An output without a gradient arrives as None; its backbone's parameters then
    get None and, like a backbone whose parameters and image need no gradient, its backward launches nothing."""

    @staticmethod
    def forward(ctx, img, module, *params):
        h, outs, saved = module._forward_train(img, params, True)
        ctx.set_materialize_grads(False)
        ctx.handle, ctx.module, ctx.dtype, ctx.B = h, module, img.dtype, img.shape[0]
        ctx.present = [o is not None for o in outs]
        ctx.n_params = [len(list(p[0].encoder.parameters())) + 2 if p is not None else 0 for p in module._parts()]
        ctx.save_for_backward(_lib.dev_f32(img, "img"), saved, *params)
        return tuple(o for o in outs if o is not None)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        x, saved, *params = ctx.saved_tensors
        m, dev, B = ctx.module, saved.device, ctx.B
        it = iter(grads)
        g = [next(it) if p else None for p in ctx.present]
        g = [None if t is None else _lib.dev_f32(t, "grad") for t in g]
        args, keep, _ = m._train_args(dev, params)
        gr = _lib.SmkEncoderTrainGrads()
        out, j = [], 0
        for i, n in enumerate(ctx.n_params):
            if n == 0:
                continue
            mine = []
            for k in range(n):
                want = g[i] is not None and ctx.needs_input_grad[2 + j + k]
                mine.append(torch.empty_like(params[j + k]) if want else None)
            ptrs = [None] * (5 * ((n - 2) // 3))
            for c in range(n - 2):            # parameter c of the backbone is tensor 5 * (c // 3) + c % 3
                ptrs[5 * (c // 3) + c % 3] = mine[c]
            arr = (_lib.c_f32p * len(ptrs))(*[C.cast(t.data_ptr(), _lib.c_f32p) if t is not None else None for t in ptrs])
            keep.append(arr)
            gr.tensors[i] = C.cast(arr, C.POINTER(_lib.c_f32p))
            gr.head_w[i] = C.cast(mine[-2].data_ptr(), _lib.c_f32p) if mine[-2] is not None else None
            gr.head_b[i] = C.cast(mine[-1].data_ptr(), _lib.c_f32p) if mine[-1] is not None else None
            out += mine
            j += n
        g_img = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        ws = m._native_workspace("train", _lib.call("smk_encoder_train_workspace_bytes", dev, ctx.handle, B), dev)
        _lib.call("smk_encoder_backward_train", dev, ctx.handle, C.byref(args), x, B, saved, saved.numel() * 4, *g, g_img,
                  C.byref(gr), ws, ws.numel())
        return (None if g_img is None else g_img.to(ctx.dtype), None, *out)


class PoseEncoder(_NativeEncoder):
    def __init__(self):
        super().__init__()
        self.encoder, feature_dim = create_backbone("tf_mobilenetv3_small_minimal_100")
        self.pose_cam_layers = nn.Sequential(nn.Linear(feature_dim, 6))
        self._init_native()
        self.init_weights()

    def init_weights(self):                     # smirk_encoder.py:26-31
        self.pose_cam_layers[-1].weight.data *= 0.001
        self.pose_cam_layers[-1].bias.data *= 0.001
        self.pose_cam_layers[-1].weight.data[3] = 0
        self.pose_cam_layers[-1].bias.data[3] = 7

    def _parts(self):
        return ((self, self.pose_cam_layers[0]), None, None)

    def forward(self, img):                     # smirk_encoder.py:34-45
        pose_cam = self._run(img)[0]
        return {"pose_params": pose_cam[..., :3], "cam": pose_cam[..., 3:]}


class ShapeEncoder(_NativeEncoder):
    def __init__(self, n_shape=300):
        super().__init__()
        self.encoder, feature_dim = create_backbone("tf_mobilenetv3_large_minimal_100")
        self.shape_layers = nn.Sequential(nn.Linear(feature_dim, n_shape))
        self._init_native(n_shape=n_shape)
        self.init_weights()

    def init_weights(self):                     # smirk_encoder.py:61-63
        self.shape_layers[-1].weight.data *= 0
        self.shape_layers[-1].bias.data *= 0

    def _parts(self):
        return (None, (self, self.shape_layers[0]), None)

    def forward(self, img):                     # smirk_encoder.py:66-73
        return {"shape_params": self._run(img)[1]}


class ExpressionEncoder(_NativeEncoder):
    def __init__(self, n_exp=50):
        super().__init__()
        self.encoder, feature_dim = create_backbone("tf_mobilenetv3_large_minimal_100")
        self.expression_layers = nn.Sequential(nn.Linear(feature_dim, n_exp + 2 + 3))
        self._init_native(n_exp=n_exp)
        self.init_weights()

    def init_weights(self):                     # smirk_encoder.py:90-92
        self.expression_layers[-1].weight.data *= 0.1
        self.expression_layers[-1].bias.data *= 0.1

    def _parts(self):
        return (None, None, (self, self.expression_layers[0]))

    def forward(self, img):                     # smirk_encoder.py:95-110 (clamps applied by the native head kernel)
        expr, ne = self._run(img)[2], self.n_exp
        return {"expression_params": expr[..., :ne], "eyelid_params": expr[..., ne:ne + 2], "jaw_params": expr[..., ne + 2:ne + 5]}


class SmirkEncoder(_NativeEncoder):
    def __init__(self, n_exp=50, n_shape=300):
        super().__init__()
        self.pose_encoder = PoseEncoder()
        self.shape_encoder = ShapeEncoder(n_shape=n_shape)
        self.expression_encoder = ExpressionEncoder(n_exp=n_exp)
        self._init_native(n_exp=n_exp, n_shape=n_shape)

    def _parts(self):
        return ((self.pose_encoder, self.pose_encoder.pose_cam_layers[0]),
                (self.shape_encoder, self.shape_encoder.shape_layers[0]),
                (self.expression_encoder, self.expression_encoder.expression_layers[0]))

    def forward(self, img):                     # smirk_encoder.py:123-133: one native call runs the three backbones concurrently
        pose_cam, shape, expr = self._run(img)
        ne = self.n_exp
        return {
            "pose_params": pose_cam[..., :3], "cam": pose_cam[..., 3:],
            "shape_params": shape,
            "expression_params": expr[..., :ne], "eyelid_params": expr[..., ne:ne + 2],
            "jaw_params": expr[..., ne + 2:ne + 5],
        }
