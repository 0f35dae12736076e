"""``SmirkGenerator`` — drop-in for the reference ``src/smirk_generator.py`` (eval BN).

Same constructor, sub-module names (``state_dict`` keys such as ``encoder1.enc1conv1.weight``,
``resnet_blocks.0.conv_block.1.weight``, ``upconv4.bias``) and forward signature.  The torch modules are
parameter containers; the forward pass runs in ``csrc/generator.cu`` through ``smk_generator_forward``.

With grad mode on and an input that requires grad, a frozen (``requires_grad_(False)``) eval-mode generator passes the
gradient to its input, as the reference trainer's emotion loss and photometric fitting need: the forward then keeps
its activations (``smk_generator_forward_saved``) and the backward runs ``smk_generator_backward``.  Eval-mode weight
gradients are not implemented.

Train mode (``.train()``, what the reference trainer's generator steps run) is opt-in, as the encoder's: per module with
``allow_train_mode_(True)``, or process-wide with ``smirk_encoder.set_train_mode_default(True)`` (one flag for both
modules; ``python -m smirk_b200.dropin --train``).  Then the BatchNorms normalise with batch statistics and update their
running statistics (``smk_generator_forward_train``, also under ``torch.no_grad()``), and every parameter that requires
grad, and the input when it requires grad, gets its gradient (``smk_generator_backward_train``).  Batch statistics couple
the images of a batch.  Without the opt-in a train-mode generator raises.

Live weights (``live_weights_(True)``, off by default) run the eval path on a handle refreshed on the device from the
module's own tensors at every call (``smk_generator_refresh``), as the encoder's: for a frozen generator whose weights
another path keeps training.  Fixed inference weights keep the host-packed handle.

``precision`` (part of the native handle's key, so it may change between calls): 0 = fp32 CUDA cores, 1 = TF32 tensor cores,
3 = 3xTF32 tensor cores (each operand split into a TF32 head and tail, three products per term: fp32-equivalent forward and
input gradient, the same launches as 1).  Precisions 1 and 3 need ``init_features % 32 == 0``.
"""
import ctypes as C
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib


class ResnetBlock(nn.Module):
    """Parameter layout of smirk_generator.py:121-171 (indices 1,2 / 5,6 of ``conv_block``)."""

    def __init__(self, dim, padding_type="reflect", norm_layer=nn.BatchNorm2d, use_dropout=False, use_bias=False):
        super().__init__()
        if padding_type != "reflect" or use_dropout:
            raise NotImplementedError("smirk_b200.ResnetBlock: only reflect padding without dropout (as built at smirk_generator.py:25)")
        self.conv_block = nn.Sequential(
            nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, 3, padding=0, bias=use_bias), norm_layer(dim), nn.ReLU(True),
            nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, 3, padding=0, bias=use_bias), norm_layer(dim))


class SmirkGenerator(_lib.NativeModule, nn.Module):
    def __init__(self, in_channels=3, out_channels=1, init_features=16, res_blocks=3):
        super().__init__()
        f = init_features
        self.encoder1 = SmirkGenerator._block(in_channels, f, name="enc1")
        self.pool1 = nn.MaxPool2d(kernel_size=2, stride=2)
        self.encoder2 = SmirkGenerator._block(f, f * 2, name="enc2")
        self.pool2 = nn.MaxPool2d(kernel_size=2, stride=2)
        self.encoder3 = SmirkGenerator._block(f * 2, f * 4, name="enc3")
        self.pool3 = nn.MaxPool2d(kernel_size=2, stride=2)
        self.encoder4 = SmirkGenerator._block(f * 4, f * 8, name="enc4")
        self.pool4 = nn.MaxPool2d(kernel_size=2, stride=2)
        self.bottleneck = SmirkGenerator._block(f * 8, f * 16, name="bottleneck")
        self.resnet_blocks = nn.ModuleList([ResnetBlock(f * 16) for _ in range(res_blocks)])
        self.upconv4 = nn.ConvTranspose2d(f * 16, f * 8, kernel_size=2, stride=2)
        self.decoder4 = SmirkGenerator._block(f * 16, f * 8, name="dec4")
        self.upconv3 = nn.ConvTranspose2d(f * 8, f * 4, kernel_size=2, stride=2)
        self.decoder3 = SmirkGenerator._block(f * 8, f * 4, name="dec3")
        self.upconv2 = nn.ConvTranspose2d(f * 4, f * 2, kernel_size=2, stride=2)
        self.decoder2 = SmirkGenerator._block(f * 4, f * 2, name="dec2")
        self.upconv1 = nn.ConvTranspose2d(f * 2, f, kernel_size=2, stride=2)
        self.decoder1 = SmirkGenerator._block(f * 2, f, name="dec1")
        self.conv = nn.Conv2d(in_channels=f, out_channels=out_channels, kernel_size=1)
        self._cfg = (in_channels, out_channels, init_features, res_blocks)
        self.precision = 0

    @staticmethod
    def _block(in_channels, features, name):
        return nn.Sequential(OrderedDict([
            (name + "conv1", nn.Conv2d(in_channels, features, kernel_size=3, padding=1, bias=False)),
            (name + "norm1", nn.BatchNorm2d(num_features=features)),
            (name + "relu1", nn.ReLU(inplace=True)),
            (name + "conv2", nn.Conv2d(features, features, kernel_size=3, padding=1, bias=False)),
            (name + "norm2", nn.BatchNorm2d(num_features=features)),
            (name + "relu2", nn.ReLU(inplace=True)),
        ]))

    def _native_extras(self):
        return (self.precision,)

    def _native_create(self, device):
        keep = []
        ts = [v for k, v in self.state_dict().items() if not k.endswith("num_batches_tracked")]
        arr = (_lib.c_f32p * len(ts))()
        for j, t in enumerate(ts):
            a, p = _lib.f32(t)
            keep.append(a)
            arr[j] = p
        d = _lib.SmkGeneratorDesc()
        d.in_channels, d.out_channels, d.init_features, d.res_blocks = self._cfg
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(_lib.c_f32p)), len(ts), self.precision
        return _lib.create("generator", d, device)

    def _check_input(self, x):
        cin = self._cfg[0]
        if x.dim() != 4 or tuple(x.shape[1:]) != (cin, 224, 224):
            raise RuntimeError("smirk_b200.SmirkGenerator: expected x [B,%d,224,224], got %s" % (cin, tuple(x.shape)))

    def allow_train_mode_(self, on=True):
        """Opt this module in to (or out of) train mode; returns the module."""
        self._allow_train = bool(on)
        return self

    def live_weights_(self, on=True):
        """Run the eval path on weights refreshed on the device at every call (see the module docstring); returns the
        module."""
        self._live = bool(on)
        return self

    def _live_tensors(self):
        """The tensors a refresh reads: the state_dict's in its order, without num_batches_tracked."""
        return [v for k, v in self.state_dict(keep_vars=True).items() if not k.endswith("num_batches_tracked")]

    def _refresh(self, h, dev, tensors):
        """smk_generator_refresh of live handle h from ``_live_tensors()`` (or the tensors an autograd context saved)."""
        eps = {m.eps for m in self.modules() if isinstance(m, nn.BatchNorm2d)}
        if len(eps) != 1:
            raise RuntimeError("smirk_b200.SmirkGenerator: live weights need one eps for all BatchNorms, got %s" % sorted(eps))
        for t in tensors:
            if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("smirk_b200: live weights need contiguous float32 parameters and buffers on %s" % dev)
        arr = (_lib.c_f32p * len(tensors))(*[C.cast(t.data_ptr(), _lib.c_f32p) for t in tensors])
        a = _lib.SmkGeneratorTrainArgs()
        a.tensors, a.n_tensors, a.eps = C.cast(arr, C.POINTER(_lib.c_f32p)), len(tensors), eps.pop()
        _lib.refresh("generator", h, dev, a)

    def _eval_handle(self, dev):
        """-> (handle, tensors): the host-packed eval handle and None, or with live weights the live handle (keyed on the
        configuration and precision only), refreshed from the tensors returned."""
        if not self.__dict__.get("_live"):
            return self._native_handle(dev), None
        h = _lib.live_handle(self, "generator", dev, (self._cfg, int(self.precision)), self._cfg + (int(self.precision),))
        tensors = self._live_tensors()
        self._refresh(h, dev, tensors)
        return h, tensors

    def _train_allowed(self):
        on = self.__dict__.get("_allow_train")
        return _lib.train_mode_default() if on is None else on

    def _is_train(self):
        """True when the BatchNorms are in train mode (checked on every call: .train() after the first forward must not
        silently run eval BN)."""
        modes = {m.training for m in self.modules() if isinstance(m, nn.BatchNorm2d)}
        if True not in modes:
            return False
        if not self._train_allowed():
            raise RuntimeError("smirk_b200.SmirkGenerator: train-mode BatchNorm runs only with the opt-in: call "
                               ".allow_train_mode_(True) on the generator or run under `python -m smirk_b200.dropin --train`")
        if modes != {True}:
            raise RuntimeError("smirk_b200.SmirkGenerator: its BatchNorms mix train and eval mode")
        return True

    def forward(self, x):
        _lib.require_cuda(x, "x")
        if self._is_train():
            self._check_input(x)
            return self._run_train(x)
        if torch.is_grad_enabled() and x.requires_grad:
            if any(p.requires_grad for p in self.parameters()):
                raise RuntimeError("smirk_b200.SmirkGenerator: weight gradients are not implemented; to pass a gradient to the "
                                   "input, freeze the generator with .requires_grad_(False)")
            self._check_input(x)
            return _GeneratorFunction.apply(x, self)
        with torch.no_grad():
            dev = x.device
            h = self._eval_handle(dev)[0]
            x = _lib.dev_f32(x, "x")
            self._check_input(x)
            B = x.shape[0]
            y = torch.empty(B, self._cfg[1], 224, 224, dtype=torch.float32, device=dev)
            ws = self._native_workspace("forward", _lib.call("smk_generator_workspace_bytes", dev, h, B), dev)
            _lib.call("smk_generator_forward", dev, h, x, B, y, ws, ws.numel())
            return y

    def _forward_saved(self, x):
        """-> (handle, outputs, saved) of ``_forward_saved_live``."""
        return self._forward_saved_live(x)[:3]

    def _forward_saved_live(self, x):
        """-> (handle, y, saved, live tensors | None): the grad-mode forward, its activations in a buffer of their own."""
        dev = x.device
        h, tensors = self._eval_handle(dev)
        x = _lib.dev_f32(x, "x")
        B = x.shape[0]
        y = torch.empty(B, self._cfg[1], 224, 224, dtype=torch.float32, device=dev)
        saved = _lib.saved_buffer("generator", h, B, dev)
        ws = self._native_workspace("forward", _lib.call("smk_generator_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_generator_forward_saved", dev, h, x, B, y, saved, saved.numel() * 4, ws, ws.numel())
        return h, y, saved, tensors

    @torch.no_grad()
    def saved_activations(self, x):
        """The activations the backward of ``self(x)`` uses, {reference layer name: [B,C,H,W] tensor}: the post-ReLU
        output of every block conv (``enc1conv1`` ... ``dec1conv2``) and of every ResNet block's first conv
        (``res0conv1`` ...).  The forward is deterministic and batch-independent, so these are the tensors an autograd
        context of the same input holds."""
        _lib.require_cuda(x, "x")
        self._check_input(x)
        if self._is_train():                 # train mode: on copies of the running statistics, which stay untouched
            h, _, saved = self._forward_train(x, list(self.parameters()), True, copy_stats=True)
        else:
            h, _, saved = self._forward_saved(x)
        return _lib.saved_views("generator", h, saved, x.shape[0])

    # ---- train mode ---------------------------------------------------------------------------------------------------
    def _train_handle(self, dev):
        st = self._native
        key = (str(dev), self._cfg, int(self.precision))          # topology only: an optimizer step builds nothing
        if st.train_handle is None or st.train_key != key:
            st.train_handle = None
            h = C.c_void_p()
            _lib.call("smk_generator_train_create", dev, *self._cfg, int(self.precision), C.byref(h))
            st.train_handle, st.train_key = _lib.NativeHandle(h, "smk_generator_destroy"), key
        return st.train_handle

    def _bn_settings(self):
        bns = [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)]
        settings = {(m.momentum, m.eps) for m in bns}
        if len(settings) != 1 or not all(m.affine and m.track_running_stats for m in bns):
            raise RuntimeError("smirk_b200.SmirkGenerator: train mode needs affine BatchNorms that track running statistics, "
                               "with one momentum and one eps, got %s" % sorted(settings, key=str))
        momentum, eps = settings.pop()
        if (momentum is not None and not 0.0 <= momentum <= 1.0) or not eps > 0:
            raise RuntimeError("smirk_b200.SmirkGenerator: train mode takes momentum in [0, 1] or None and eps > 0, got "
                               "momentum %r, eps %r" % (momentum, eps))
        return momentum, eps

    def _train_args(self, dev, params, copy_stats=False):
        """-> (SmkGeneratorTrainArgs, keep-alive list, [running statistics and counters], {parameter index: tensor
        index}).  params: ``list(self.parameters())`` (or the tensors an autograd context saved).  copy_stats: point at
        copies of the running statistics (a forward that must leave the module untouched)."""
        momentum, eps = self._bn_settings()
        names = [k for k, _ in self.named_parameters()]
        it = iter(params)
        ts, nbt, stats, where = [], [], [], {}
        for k, v in self.state_dict(keep_vars=True).items():
            if k.endswith("num_batches_tracked"):
                n = v.clone() if copy_stats else v
                if n.device != dev or n.dtype != torch.int64:
                    raise RuntimeError("smirk_b200: num_batches_tracked must be an int64 tensor on %s" % dev)
                nbt.append(n); stats.append(n)
                continue
            if k in names:
                where[names.index(k)] = len(ts)
                t = next(it)
            else:
                t = v.clone() if copy_stats else v
                stats.append(t)
            if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("smirk_b200: train mode needs contiguous float32 parameters and buffers on %s" % dev)
            ts.append(t)
        a = _lib.SmkGeneratorTrainArgs()
        arr = (_lib.c_f32p * len(ts))(*[C.cast(t.data_ptr(), _lib.c_f32p) for t in ts])
        narr = (C.POINTER(C.c_int64) * len(nbt))(*[C.cast(t.data_ptr(), C.POINTER(C.c_int64)) for t in nbt])
        a.tensors, a.n_tensors = C.cast(arr, C.POINTER(_lib.c_f32p)), len(ts)
        a.num_batches_tracked = C.cast(narr, C.POINTER(C.POINTER(C.c_int64)))
        a.momentum, a.eps = -1.0 if momentum is None else momentum, eps
        return a, [arr, narr, ts, nbt], stats, where

    def _forward_train(self, x, params, with_saved, copy_stats=False):
        """-> (handle, y, saved | None): one train-mode forward, which updates the running statistics (of copies, with
        copy_stats)."""
        dev = x.device
        h = self._train_handle(dev)
        x = _lib.dev_f32(x, "x")
        B = x.shape[0]
        y = torch.empty(B, self._cfg[1], 224, 224, dtype=torch.float32, device=dev)
        args, keep, stats, _ = self._train_args(dev, params, copy_stats)
        nbytes = _lib.call("smk_generator_train_workspace_bytes", dev, h, B)
        saved = _lib.saved_buffer("generator", h, B, dev) if with_saved else None
        if saved is None:
            nbytes += _lib.call("smk_generator_saved_bytes", dev, h, B)
        ws = self._native_workspace("train", nbytes, dev)
        _lib.call("smk_generator_forward_train", dev, h, C.byref(args), x, B, y, saved, 0 if saved is None else saved.numel() * 4,
                  ws, ws.numel())
        if not copy_stats:                  # the eval handle repacks, and copies see the new statistics
            for t in stats:
                torch.autograd.graph.increment_version(t)
        return h, y, saved

    def _run_train(self, x):
        params = list(self.parameters())
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
            return _GeneratorTrainFunction.apply(x, self, *params)
        with torch.no_grad():
            return self._forward_train(x, params, False)[1]


class _GeneratorFunction(torch.autograd.Function):
    """Frozen generator: y = G(x), and the gradient with respect to x only.  The activations are saved per call, so
    several forwards may share one backward.  With live weights the tensors the refresh read are saved too (autograd
    raises if one is modified in place before the backward), and the backward refreshes the handle from them again when
    another call has refreshed it since."""

    @staticmethod
    def forward(ctx, x, module):
        h, y, saved, tensors = module._forward_saved_live(x)
        ctx.handle, ctx.module, ctx.dtype = h, module, x.dtype    # the handle the activations were computed with
        ctx.live = tensors is not None
        ctx.generation = h.generation if ctx.live else None
        ctx.save_for_backward(y, saved, *(tensors or ()))
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_y):
        y, saved, *tensors = ctx.saved_tensors
        m, dev, B = ctx.module, y.device, y.shape[0]
        if ctx.live and ctx.handle.generation != ctx.generation:
            m._refresh(ctx.handle, dev, tensors)
            ctx.generation = ctx.handle.generation
        g_y = _lib.dev_f32(g_y, "g_y")
        g_x = torch.empty(B, m._cfg[0], 224, 224, dtype=torch.float32, device=dev)
        ws = m._native_workspace("backward", _lib.call("smk_generator_backward_workspace_bytes", dev, ctx.handle, B), dev)
        _lib.call("smk_generator_backward", dev, ctx.handle, B, y, saved, saved.numel() * 4, g_y, g_x, ws, ws.numel())
        return g_x.to(ctx.dtype), None


class _GeneratorTrainFunction(torch.autograd.Function):
    """Train-mode generator: y = G(x), and the gradients of x and of every parameter in ``parameters()`` order (those
    autograd asks for).  The activations and batch statistics are saved per call, so several forwards may share one
    backward."""

    @staticmethod
    def forward(ctx, x, module, *params):
        h, y, saved = module._forward_train(x, params, True)
        ctx.handle, ctx.module, ctx.dtype = h, module, x.dtype
        ctx.save_for_backward(y, saved, *params)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_y):
        y, saved, *params = ctx.saved_tensors
        m, dev, B = ctx.module, y.device, y.shape[0]
        g_y = _lib.dev_f32(g_y, "g_y")
        args, keep, _, where = m._train_args(dev, params)
        out = [torch.empty_like(p) if ctx.needs_input_grad[2 + i] else None for i, p in enumerate(params)]
        ptrs = [None] * args.n_tensors
        for i, t in enumerate(out):
            ptrs[where[i]] = t
        arr = (_lib.c_f32p * len(ptrs))(*[C.cast(t.data_ptr(), _lib.c_f32p) if t is not None else None for t in ptrs])
        gr = _lib.SmkGeneratorTrainGrads()
        gr.tensors = C.cast(arr, C.POINTER(_lib.c_f32p))
        g_x = torch.empty(B, m._cfg[0], 224, 224, dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        ws = m._native_workspace("train", _lib.call("smk_generator_train_workspace_bytes", dev, ctx.handle, B), dev)
        _lib.call("smk_generator_backward_train", dev, ctx.handle, C.byref(args), B, y, saved, saved.numel() * 4, g_y, g_x,
                  C.byref(gr), ws, ws.numel())
        return (None if g_x is None else g_x.to(ctx.dtype), None, *out)
