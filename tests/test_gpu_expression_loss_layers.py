"""The expression loss's own kernels one at a time against float64, through the kernel-test entry points
smk_debug_expression_* (csrc/expression_loss.cu), and the convolution problems no other network runs through
smk_debug_mica_conv.

- Small-integer data makes every sum exact in fp32: the stem im2col, the max pool (with ties: the first maximum wins),
  its backward, the stride-2 col2im and the stem dgrad must equal float64 bit for bit.
- Random data stays within a stated bound: (1024 + 16) 2^-24 S for the stem dgrad (S: the sum of the magnitudes of its
  terms), 2^-20 to 2^-18 relative for the head, and
  |out - ref| <= (K + 16) 2^-22 S (S = |scale| sum_k |a w| + |bias| + |res|) for the convolutions, as in
  test_gpu_mica_layers.py.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
_vp, _i = C.c_void_p, C.c_int


@pytest.fixture(scope="module")
def L(native_lib):
    sig = {"im2col": [_vp, _vp, _i, _i, _vp, _vp], "maxpool": [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp],
           "maxpool_bwd": [_vp, _vp, _i, _i, _i, _vp, _vp], "col2im": [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp],
           "stem_dgrad": [_vp, _vp, _i, _i, _vp, _vp, _vp], "head": [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp],
           "head_bwd": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]}
    for k, a in sig.items():
        fn = getattr(native_lib, "smk_debug_expression_" + k)
        fn.restype, fn.argtypes = _i, a
    native_lib.smk_debug_mica_conv.restype = _i
    native_lib.smk_debug_mica_conv.argtypes = [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp,
                                               _vp, _i, _i, _vp, _i, _vp, _vp, _i, _vp]
    return native_lib


def call(L, name, *args):
    s = torch.cuda.current_stream().cuda_stream
    args = [a.data_ptr() if torch.is_tensor(a) else a for a in args]
    rc = getattr(L, name)(*args, s)
    assert rc == 0, L.smk_last_error()
    torch.cuda.synchronize()


def ints(g, *shape, lo=-2, hi=3):
    return torch.randint(lo, hi, shape, generator=g).float()


def test_stem_im2col(L):
    g = torch.Generator().manual_seed(1)
    B = 2
    a, b = torch.rand(B, 3, 224, 224, generator=g), torch.rand(B, 3, 224, 224, generator=g)
    out = torch.empty(2 * B * 112 * 112, 148, device=DEV)
    call(L, "smk_debug_expression_im2col", a.to(DEV), b.to(DEV), B, 0, out)
    x = torch.cat([a, b])
    cols = F.unfold(x, 7, padding=3, stride=2).view(2 * B, 3, 49, 112 * 112)           # [img, c, tap, pix]
    ref = torch.zeros(2 * B, 112 * 112, 148)
    ref[:, :, :147] = cols.permute(0, 3, 2, 1).reshape(2 * B, 112 * 112, 147)          # k = tap * 3 + c
    assert torch.equal(out.cpu().view(2 * B, 112 * 112, 148), ref)
    call(L, "smk_debug_expression_im2col", a.to(DEV), b.to(DEV), B, 1, out)
    rna = ((ref.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    assert torch.equal(out.cpu().view(2 * B, 112 * 112, 148), rna)


@pytest.mark.parametrize("H,C", [(112, 64), (9, 8)])
def test_maxpool_first_maximum_and_backward(L, H, C):
    g = torch.Generator().manual_seed(H)
    Bi, save = 3, 2
    x = ints(g, Bi, H, H, C, lo=0, hi=3)                  # many ties
    Ho = (H + 1) // 2
    out, out2 = torch.empty(Bi, Ho, Ho, C, device=DEV), torch.empty(save, Ho, Ho, C, device=DEV)
    arg = torch.empty(save, Ho, Ho, C, dtype=torch.int8, device=DEV)
    call(L, "smk_debug_expression_maxpool", x.to(DEV), Bi, H, C, out, save, out2, arg)
    rv, ri = F.max_pool2d(x.permute(0, 3, 1, 2).double(), 3, 2, 1, return_indices=True)
    assert torch.equal(out.cpu().double(), rv.permute(0, 2, 3, 1)) and torch.equal(out2.cpu(), out[:save].cpu())
    h, w = ri // H, ri % H
    oh, ow = torch.arange(Ho).view(1, 1, Ho, 1), torch.arange(Ho).view(1, 1, 1, Ho)
    tap = ((h - 2 * oh + 1) * 3 + (w - 2 * ow + 1)).permute(0, 2, 3, 1)
    assert torch.equal(arg.cpu().long(), tap[:save])
    gp = ints(g, save, Ho, Ho, C)
    gin = torch.empty(save, H, H, C, device=DEV)
    call(L, "smk_debug_expression_maxpool_bwd", gp.to(DEV), arg, save, H, C, gin)
    xl = x[:save].permute(0, 3, 1, 2).double().requires_grad_()
    ref, = torch.autograd.grad(F.max_pool2d(xl, 3, 2, 1), [xl], gp.permute(0, 3, 1, 2).double())
    assert torch.equal(gin.cpu().double(), ref.permute(0, 2, 3, 1))


def gather_ref(x, taps):
    """The gather of smk::gather_s2 in float64: x [B,H,H,C] -> [B*(H/2)^2, taps*C]."""
    B, H, _, C = x.shape
    if taps == 1:
        return x[:, ::2, ::2, :].reshape(-1, C)
    cols = F.unfold(x.permute(0, 3, 1, 2), 3, padding=1, stride=2).view(B, C, 9, -1)
    return cols.permute(0, 3, 2, 1).reshape(-1, 9 * C)


@pytest.mark.parametrize("Ho,C,taps", [(28, 128, 9), (14, 256, 9), (7, 512, 9), (28, 256, 1), (7, 1024, 1)])
def test_col2im_is_the_gathers_adjoint(L, Ho, C, taps):
    g = torch.Generator().manual_seed(Ho * C + taps)
    Bi = 2
    dg = ints(g, Bi * Ho * Ho, taps * C)
    mask = ints(g, Bi, 2 * Ho, 2 * Ho, C, lo=-1, hi=2)
    x = torch.zeros(Bi, 2 * Ho, 2 * Ho, C, dtype=torch.float64, requires_grad=True)
    ref, = torch.autograd.grad(gather_ref(x, taps), [x], dg.double())
    for m, r in ((None, ref), (mask, ref * (mask > 0))):
        out = torch.empty(Bi, 2 * Ho, 2 * Ho, C, device=DEV)
        call(L, "smk_debug_expression_col2im", dg.to(DEV), Bi, Ho, C, taps, None if m is None else m.to(DEV), 0, out)
        assert torch.equal(out.cpu().double(), r)


@pytest.mark.parametrize("integer", [True, False])
def test_stem_dgrad(L, integer):
    g = torch.Generator().manual_seed(5)
    B, Bi = 1, 2
    if integer:
        gs, wd = ints(g, Bi, 112, 112, 64), ints(g, 147, 64)
    else:
        gs, wd = torch.randn(Bi, 112, 112, 64, generator=g), torch.randn(147, 64, generator=g) * 0.1
    o0, o1 = torch.empty(B, 3, 224, 224, device=DEV), torch.empty(Bi - B, 3, 224, 224, device=DEV)
    call(L, "smk_debug_expression_stem_dgrad", gs.to(DEV), wd.to(DEV), B, Bi, o0, o1)
    w = wd.double().view(7, 7, 3, 64).permute(3, 2, 0, 1)                              # [co][c][ky][kx]
    ref = F.conv_transpose2d(gs.permute(0, 3, 1, 2).double(), w, stride=2, padding=3, output_padding=1)
    got = torch.cat([o0, o1]).cpu().double()
    if integer:
        assert torch.equal(got, ref)
    else:                                              # <= 16 taps x 64 channels = 1024 fp32 terms per output
        S = F.conv_transpose2d(gs.permute(0, 3, 1, 2).double().abs(), w.abs(), stride=2, padding=3, output_padding=1)
        assert bool(((got - ref).abs() <= (1024 + 16) * 2.0 ** -24 * S).all())


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("use_mean", [0, 1])
def test_head_forward_and_backward(L, metric, use_mean):
    g = torch.Generator().manual_seed(10 + metric)
    B = 3
    y = torch.rand(2 * B, 7, 7, 2048, generator=g) - 0.3
    y = y.clamp_min(0)
    feat, lossv = torch.empty(2 * B, 2048, device=DEV), torch.empty(B, device=DEV)
    loss = torch.empty(() if use_mean else (B,), device=DEV)
    for swap in (0, 1):
        call(L, "smk_debug_expression_head", y.to(DEV), B, swap, metric, use_mean, feat, lossv, loss)
        yd = y.double().requires_grad_()
        f = yd.mean(dim=(1, 2))
        fg, ft = (f[B:], f[:B]) if swap else (f[:B], f[B:])
        ref = [((fg - ft) ** 2).mean(1), (fg - ft).abs().mean(1), 1 - F.cosine_similarity(fg, ft, dim=1)][metric]
        ref = ref.mean() if use_mean else ref
        assert float((feat.cpu().double() - torch.cat([fg, ft]).detach()).abs().max()) <= 2 ** -20 * float(f.detach().abs().max())
        assert float((loss.cpu().double() - ref.detach()).abs().max()) <= 2 ** -18 * float(ref.detach().abs().max())
    up = torch.rand(() if use_mean else (B,), generator=g) + 0.5
    yd = y.double().requires_grad_()
    f = yd.mean(dim=(1, 2))
    ref = [((f[:B] - f[B:]) ** 2).mean(1), (f[:B] - f[B:]).abs().mean(1), 1 - F.cosine_similarity(f[:B], f[B:], dim=1)][metric]
    ref = ref.mean() if use_mean else ref
    gy, = torch.autograd.grad(ref, [yd], up.double())
    call(L, "smk_debug_expression_head", y.to(DEV), B, 0, metric, use_mean, feat, lossv, loss)
    out = torch.empty(2 * B, 7, 7, 2048, device=DEV)
    call(L, "smk_debug_expression_head_bwd", feat, y.to(DEV), up.to(DEV), B, 2 * B, 0, metric, use_mean, 0, out)
    gy = gy * (y > 0)
    assert float((out.cpu().double() - gy).abs().max()) <= 2 ** -18 * float(gy.abs().max())
    out1 = torch.empty(B, 7, 7, 2048, device=DEV)          # tar alone (swap): the first B chain images are tar's
    call(L, "smk_debug_expression_head_bwd", feat, y[B:].to(DEV).contiguous(), up.to(DEV), B, B, 1, metric, use_mean, 0, out1)
    assert float((out1.cpu().double() - gy[B:]).abs().max()) <= 2 ** -18 * float(gy.abs().max())


# (name, rows per image, K, N): the GEMM problems only this network issues, as plain GEMMs over [M, K] operands
CONVS = [("stem", 112 * 112, 148, 64), ("layer4_conv1", 49, 2048, 512), ("layer4_conv3", 49, 512, 2048),
         ("layer3_ds_s2", 196, 512, 1024), ("layer4_ds_s2", 49, 1024, 2048), ("layer2_conv2_s2", 784, 1152, 128),
         ("layer3_conv2_s2", 196, 2304, 256), ("layer4_conv2_s2", 49, 4608, 512)]


@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("spec", CONVS, ids=[c[0] for c in CONVS])
def test_network_gemms(L, spec, precision):
    name, rows, K, N = spec
    g = torch.Generator().manual_seed(K + N)
    M = 2 * rows
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) * (2.0 / K) ** 0.5
    scale, bias, res = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1, torch.randn(M, N, generator=g)
    rna = lambda t: ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)    # noqa: E731
    if precision == 1:
        x = rna(x)
    hi = rna(w) if precision else None
    lo = rna(w - hi) if precision == 3 else None
    wk = None if precision else w.t().contiguous()
    out = torch.empty(M, N, device=DEV)
    d = lambda t: None if t is None else t.to(DEV)                                   # noqa: E731
    xs, res_d = d(x), d(res)
    call(L, "smk_debug_mica_conv", xs, K, 1, 1, M, K, d(wk), d(hi), d(lo), d(scale), d(bias), N, K, 0, res_d, N, None, out, N, 0,
         None, 0, None, None, 0)
    wr = (hi if precision == 1 else w).double()
    ref = scale.double() * (x.double() @ wr.t()) + bias.double() + res.double()
    S = scale.double() * (x.double().abs() @ wr.abs().t()) + bias.double().abs() + res.double().abs()
    bound = (K + 16) * 2.0 ** -22 * S
    if precision == 1:
        bound = bound + (K + 16) * 2.0 ** -22 * S                  # the TF32 product of TF32 operands, fp32 sums
    err = (out.cpu().double() - ref).abs()
    print("%s precision %d: max err / bound %.3f" % (name, precision, float((err / bound).max())))
    assert bool((err <= bound).all())
