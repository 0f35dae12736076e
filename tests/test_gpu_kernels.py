"""GPU suite (-m gpu): single convolution kernels through the C ABI's test entry points against
torch fp32 on the same inputs.  fp32 CUDA-core path: 1e-5 relative.  TF32 wgmma path: TF32 operand
truncation (10-bit mantissa) bounds the error at ~1e-3 of the output scale; the torch reference for
that path is computed in fp64 so the comparison isolates the kernel's own rounding."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def make_case(B, H, W, Cin, N, seed, mode):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g)
    k = 1 if mode == 0 else 3
    w = torch.randn(N, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    scale = torch.rand(N, generator=g) + 0.5
    bias = torch.randn(N, generator=g) * 0.1
    return x, w, scale, bias


def torch_conv(x, w, scale, bias, mode, relu, res=None, dtype=torch.float64):
    x, w = x.to(dtype), w.to(dtype)
    if mode == 2:
        y = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w)
    else:
        y = F.conv2d(x, w, padding=1 if mode == 1 else 0)
    y = y * scale.to(dtype).view(1, -1, 1, 1) + bias.to(dtype).view(1, -1, 1, 1)
    if res is not None:
        y = y + res.to(dtype)
    return (F.relu(y) if relu else y).float()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def w_kn(w):          # [N,Cin,k,k] -> [K][N], k = (ky*3+kx)*Cin + c
    N, Cin, k, _ = w.shape
    return w.permute(2, 3, 1, 0).reshape(k * k * Cin, N).contiguous()


def w_nk(w):          # [N,Cin,k,k] -> [N][K]
    N, Cin, k, _ = w.shape
    return w.permute(0, 2, 3, 1).reshape(N, k * k * Cin).contiguous()


@pytest.mark.parametrize("B,H,W,Cin,N,mode,relu,use_res", [
    (2, 14, 14, 64, 64, 1, 1, 0), (1, 9, 11, 16, 24, 0, 0, 1), (3, 14, 14, 32, 96, 2, 0, 1),
    (2, 28, 28, 8, 32, 1, 1, 0), (1, 7, 7, 960, 160, 0, 0, 0), (2, 56, 56, 24, 72, 0, 1, 0),
])
def test_conv_f32_kernel(native_lib, B, H, W, Cin, N, mode, relu, use_res):
    x, w, scale, bias = make_case(B, H, W, Cin, N, 11, mode)
    res = torch.randn(B, N, H, W) if use_res else None
    ref = torch_conv(x, w, scale, bias, mode, relu, res)
    xd, wd = nhwc(x).to(DEV), w_kn(w).to(DEV)
    out = torch.empty(B, H, W, N, device=DEV)
    resd = nhwc(res).to(DEV) if use_res else None
    K = wd.shape[0]
    sd, bd = scale.to(DEV), bias.to(DEV)            # keep device tensors alive across the call
    rc = native_lib.smk_debug_conv_f32(P(xd), Cin, B, H, W, Cin, P(wd), P(sd), P(bd), N, K, mode, relu,
                                       P(resd), N, P(out), N, 0, stream())
    assert rc == 0, native_lib.smk_last_error()
    got = out.permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() <= 1e-5 * ref.abs().max() + 1e-6


def run_tc(native_lib, x, w, scale, bias, mode, relu, res=None, store=0, ld_out=None, out=None):
    B, Cin, H, W = x.shape
    N = w.shape[0]
    xd = nhwc(x).to(DEV)
    if mode == 2:                                   # kernel wants a padded buffer with reflected halo
        buf = torch.zeros(B, H + 2, W + 2, Cin, device=DEV)
        buf[:, 1:-1, 1:-1] = xd
        assert native_lib.smk_debug_reflect_halo(P(buf), B, H, W, Cin, stream()) == 0
        ref_pad = nhwc(F.pad(x, (1, 1, 1, 1), mode="reflect")).to(DEV)
        assert torch.equal(buf, ref_pad)
        xd = buf
    wd = w_nk(w).to(DEV)
    K = wd.shape[1]
    if out is None:
        out = torch.full((B, H, W, N), float("nan"), device=DEV)
    resd = nhwc(res).to(DEV) if res is not None else None
    sd, bd = scale.to(DEV), bias.to(DEV)            # keep device tensors alive across the call
    rc = native_lib.smk_debug_conv_tc(P(xd), Cin, B, H, W, Cin, P(wd), P(sd), P(bd), N, K, mode, relu,
                                      P(resd), N, 0, P(out), ld_out or N, store, stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    return out


TC_CASES = [
    # B, H,  W,  Cin, N,   mode
    (1, 16, 8, 32, 32, 0),          # one exact 128-row tile, single k-block
    (2, 14, 14, 64, 64, 0),         # partial last tile (392 rows)
    (1, 9, 11, 16, 24, 0),          # K < 32 and N < BN: TMA zero-fill on both operands
    (2, 28, 28, 200, 80, 0),        # K not a multiple of 32, N > 64
    (1, 7, 7, 960, 160, 0),         # deep K, two N tiles
    (1, 16, 8, 32, 32, 1),          # 3x3, one tile
    (2, 14, 14, 64, 128, 1),        # 3x3, tiles cross rows and images, partial tail
    (3, 14, 14, 32, 96, 2),         # 3x3 over a reflection-padded buffer
    (2, 28, 28, 128, 256, 1),       # 3x3, two N tiles, 36 k-blocks (ring wraps many times)
    (2, 160, 160, 32, 32, 1),       # 3x3 persistent path: 400 tiles on 2 CTAs per SM -> CTAs own 1 or 2 tiles
    (3, 120, 120, 64, 64, 2),       # 3x3 persistent, BN = 64, reflection-padded input, 338 tiles
    (1, 300, 300, 32, 24, 1),       # 3x3 persistent, 704 tiles -> 2-3 tiles per CTA, N < BN, partial last tile
]


@pytest.mark.parametrize("B,H,W,Cin,N,mode", TC_CASES)
def test_conv_tc_kernel(native_lib, B, H, W, Cin, N, mode):
    x, w, scale, bias = make_case(B, H, W, Cin, N, 21, mode)
    res = torch.randn(B, N, H, W)
    for relu, r in ((1, None), (0, res)):
        ref = torch_conv(x, w, scale, bias, mode, relu, r)
        out = run_tc(native_lib, x, w, scale, bias, mode, relu, r)
        got = out.permute(0, 3, 1, 2).cpu()
        assert torch.isfinite(got).all(), "unwritten / NaN outputs: %d" % int((~torch.isfinite(got)).sum())
        err = (got - ref).abs().max().item()
        assert err <= 3e-3 * ref.abs().max().item(), "max err %.3g vs scale %.3g" % (err, ref.abs().max().item())


def test_conv_tc_exact_on_tf32_representable_inputs(native_lib):
    """With operands exactly representable in TF32 (small integers) the tensor-core result is exact:
    this pins the im2col addressing, swizzle and descriptor arithmetic independent of rounding."""
    g = torch.Generator().manual_seed(5)
    B, H, W, Cin, N = 2, 14, 14, 64, 64
    x = torch.randint(-3, 4, (B, Cin, H, W), generator=g).float()
    w = torch.randint(-2, 3, (N, Cin, 3, 3), generator=g).float()
    one, zero = torch.ones(N), torch.zeros(N)
    for mode in (1, 2):
        ref = torch_conv(x, w, one, zero, mode, 0)
        got = run_tc(native_lib, x, w, one, zero, mode, 0).permute(0, 3, 1, 2).cpu()
        assert torch.equal(got, ref), "%d mismatches" % int((got != ref).sum())
    x1 = torch.randint(-3, 4, (1, 40, 9, 11), generator=g).float()
    w1 = torch.randint(-2, 3, (24, 40, 1, 1), generator=g).float()
    got = run_tc(native_lib, x1, w1, torch.ones(24), torch.zeros(24), 0, 0).permute(0, 3, 1, 2).cpu()
    assert torch.equal(got, torch_conv(x1, w1, torch.ones(24), torch.zeros(24), 0, 0))


def test_conv_tc_store_modes(native_lib):
    g = torch.Generator().manual_seed(6)
    # pixel-shuffle store == ConvTranspose2d(k=2, s=2)
    B, H, W, Cin, Cout = 2, 14, 14, 64, 32
    x = torch.randint(-3, 4, (B, Cin, H, W), generator=g).float()
    wt = torch.randint(-2, 3, (Cin, Cout, 2, 2), generator=g).float()          # ConvTranspose2d weight layout
    bias = torch.randint(-2, 3, (Cout,), generator=g).float()
    ref = F.conv_transpose2d(x, wt, bias, stride=2)
    w_nk_up = wt.permute(2, 3, 1, 0).reshape(4 * Cout, Cin).contiguous()        # n = (dy*2+dx)*Cout + co
    out = torch.full((B, 2 * H, 2 * W, 2 * Cout), float("nan"), device=DEV)     # lower half of a concat buffer
    xd, wd, sd, bd = nhwc(x).to(DEV), w_nk_up.to(DEV), torch.ones(4 * Cout, device=DEV), bias.repeat(4).to(DEV)
    rc = native_lib.smk_debug_conv_tc(P(xd), Cin, B, H, W, Cin, P(wd), P(sd), P(bd), 4 * Cout, Cin, 0, 0, P(None), 0, 0,
                                      P(out), 2 * Cout, 1, stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    assert torch.equal(out[..., :Cout].permute(0, 3, 1, 2).cpu(), ref)
    assert torch.isnan(out[..., Cout:]).all()                                   # the other slice is untouched
    # padded-interior store + residual read from a padded buffer
    x, w, scale, bias = make_case(2, 14, 14, 32, 64, 8, 1)
    res = torch.randn(2, 64, 14, 14, generator=g)
    res_pad = torch.zeros(2, 16, 16, 64, device=DEV)
    res_pad[:, 1:-1, 1:-1] = nhwc(res).to(DEV)
    outp = torch.full((2, 16, 16, 64), float("nan"), device=DEV)
    wd, xd, sd, bd = w_nk(w).to(DEV), nhwc(x).to(DEV), scale.to(DEV), bias.to(DEV)
    rc = native_lib.smk_debug_conv_tc(P(xd), 32, 2, 14, 14, 32, P(wd), P(sd), P(bd), 64, 288, 1, 0,
                                      P(res_pad), 64, 1, P(outp), 64, 2, stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    ref = torch_conv(x, w, scale, bias, 1, 0, res)
    got = outp[:, 1:-1, 1:-1].permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() <= 3e-3 * ref.abs().max()
    assert torch.isnan(outp[:, 0]).all() and torch.isnan(outp[:, :, 0]).all()


# ------------------------------------------------------------------ fused expand 1x1 + depthwise 3x3
def tf_same_dw(e, wdw, stride):
    """Depthwise 3x3 with TF-'SAME' padding (timm pad_type='same'): symmetric for stride 1, bottom/right for stride 2."""
    C = e.shape[1]
    if stride == 1:
        return F.conv2d(e, wdw, padding=1, groups=C)
    return F.conv2d(F.pad(e, (0, 1, 0, 1)), wdw, stride=2, groups=C)


@pytest.mark.parametrize("B,H,Cin,mid,stride", [
    (2, 28, 40, 120, 1),        # 2x2 tiles of 14x14, two channel chunks (64 + 56), Cin not a multiple of 32
    (1, 14, 80, 200, 1),        # single tile, 4 chunks (64,64,64,8), 3 k-blocks
    (3, 56, 24, 72, 2),         # stride 2: 56 -> 28 = 4x4 tiles of 7x7
    (2, 7, 160, 960, 1),        # 7x7: tile larger than the image, 15 chunks
    (1, 112, 16, 64, 2),        # the big one: 112 -> 56, 8x8 tiles, single chunk / k-block
    (2, 20, 24, 72, 1),         # ragged tiles: 14 + 6 columns / rows (the edge role of the depthwise threads)
    (3, 30, 16, 64, 2),         # stride 2, 30 -> 15 = 7 + 7 + 1: a one-pixel edge tile; the item stride carries through x, y and image
])
def test_xdw_fused_kernel(native_lib, B, H, Cin, mid, stride):
    g = torch.Generator().manual_seed(31)
    x = torch.randn(B, Cin, H, H, generator=g)
    w1 = torch.randn(mid, Cin, 1, 1, generator=g) / Cin ** 0.5
    s1, b1 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    wd = torch.randn(mid, 1, 3, 3, generator=g) / 3.0
    s2, b2 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    dd = torch.float64
    e = F.relu(F.conv2d(x.to(dd), w1.to(dd)) * s1.to(dd).view(1, -1, 1, 1) + b1.to(dd).view(1, -1, 1, 1))
    ref = F.relu(tf_same_dw(e, wd.to(dd), stride) * s2.to(dd).view(1, -1, 1, 1) + b2.to(dd).view(1, -1, 1, 1)).float()
    Ho = (H + stride - 1) // stride
    xd, w1d = nhwc(x).to(DEV), w1.view(mid, Cin).contiguous().to(DEV)
    wdd = wd.view(mid, 9).t().contiguous().to(DEV)                      # [9][mid]
    s1d, b1d, s2d, b2d = s1.to(DEV), b1.to(DEV), s2.to(DEV), b2.to(DEV)
    out = torch.full((B, Ho, Ho, mid), float("nan"), device=DEV)
    rc = native_lib.smk_debug_xdw(P(xd), B, H, H, Cin, P(w1d), P(s1d), P(b1d), mid, P(wdd), P(s2d), P(b2d), stride, 0, P(out), stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu()
    assert torch.isfinite(got).all(), "unwritten outputs: %d" % int((~torch.isfinite(got)).sum())
    err = (got - ref).abs().max().item()
    assert err <= 3e-3 * ref.abs().max().item(), "max err %.3g vs scale %.3g" % (err, ref.abs().max().item())


def test_xdw_fused_exact_on_small_integers(native_lib):
    g = torch.Generator().manual_seed(32)
    for stride, H in ((1, 28), (2, 28)):
        B, Cin, mid = 2, 24, 72
        x = torch.randint(-2, 3, (B, Cin, H, H), generator=g).float()
        w1 = torch.randint(-1, 2, (mid, Cin, 1, 1), generator=g).float()
        wd = torch.randint(-1, 2, (mid, 1, 3, 3), generator=g).float()
        one, zero = torch.ones(mid), torch.zeros(mid)
        ref = F.relu(tf_same_dw(F.relu(F.conv2d(x, w1)), wd, stride))
        Ho = (H + stride - 1) // stride
        xd, w1d, wdd = nhwc(x).to(DEV), w1.view(mid, Cin).contiguous().to(DEV), wd.view(mid, 9).t().contiguous().to(DEV)
        od, zd = one.to(DEV), zero.to(DEV)
        out = torch.full((B, Ho, Ho, mid), float("nan"), device=DEV)
        rc = native_lib.smk_debug_xdw(P(xd), B, H, H, Cin, P(w1d), P(od), P(zd), mid, P(wdd), P(od), P(zd), stride, 0, P(out), stream())
        assert rc == 0, native_lib.smk_last_error()
        torch.cuda.synchronize()
        assert torch.equal(out.permute(0, 3, 1, 2).cpu(), ref), "stride %d" % stride


# ----------------------------------------------------------------- fused stem + block 0 (nn_kernels.cu stem_ds)
@pytest.mark.parametrize("B,H,stride", [(2, 224, 1), (2, 224, 2), (3, 64, 1), (1, 32, 2)])
def test_stem_ds_fused_kernel(native_lib, B, H, stride):
    """conv_stem 3x3 s2 (TF-SAME) + BN + ReLU -> depthwise 3x3 s{1,2} + BN + ReLU -> 1x1 16->16 + BN (+ skip at
    stride 1) against torch in float64; fp32 CUDA-core path, so the 1e-4 tolerance of the fp32 encoder applies."""
    g = torch.Generator().manual_seed(51)
    dd = torch.float64
    img = torch.rand(B, 3, H, H, generator=g)
    ws = torch.randn(16, 3, 3, 3, generator=g) / 27 ** 0.5
    wd = torch.randn(16, 1, 3, 3, generator=g) / 3.0
    wp = torch.randn(16, 16, 1, 1, generator=g) / 4.0
    sb = [(torch.rand(16, generator=g) + 0.5, torch.randn(16, generator=g) * 0.2) for _ in range(3)]
    bn = lambda t, i: t * sb[i][0].to(dd).view(1, -1, 1, 1) + sb[i][1].to(dd).view(1, -1, 1, 1)
    s = F.relu(bn(F.conv2d(F.pad(img.to(dd), (0, 1, 0, 1)), ws.to(dd), stride=2), 0))
    d = F.relu(bn(tf_same_dw(s, wd.to(dd), stride), 1))
    ref = bn(F.conv2d(d, wp.to(dd)), 2)
    if stride == 1:
        ref = ref + s
    ref = ref.float()
    Ho = H // 2 // stride
    t = [img.contiguous().to(DEV), ws.view(16, 27).t().contiguous().to(DEV), sb[0][0].to(DEV), sb[0][1].to(DEV),
         wd.view(16, 9).t().contiguous().to(DEV), sb[1][0].to(DEV), sb[1][1].to(DEV),
         wp.view(16, 16).t().contiguous().to(DEV), sb[2][0].to(DEV), sb[2][1].to(DEV)]
    out = torch.full((B, Ho, Ho, 16), float("nan"), device=DEV)
    rc = native_lib.smk_debug_stem_ds(P(t[0]), B, H, H, *[P(x) for x in t[1:]], stride, 0, P(out), stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu()
    assert torch.isfinite(got).all(), "unwritten outputs: %d" % int((~torch.isfinite(got)).sum())
    err = (got - ref).abs().max().item()
    assert err <= 1e-4 * ref.abs().max().item(), "max err %.3g vs scale %.3g" % (err, ref.abs().max().item())


# ----------------------------------------------------------------- 3xTF32 error-compensated variants (encoder precision 3)
def tf32_split(w):
    """hi = tf32(w) (round to nearest, ties away — cvt.rna), lo = tf32(w - hi): what smk_encoder_create packs."""
    def rna(t):
        u = t.contiguous().view(torch.int32)
        r = ((u + 0x1000) & ~0x1FFF).view(torch.float32)
        return r
    hi = rna(w)
    return hi, rna(w - hi)


@pytest.mark.parametrize("M,K,N,relu,use_res", [
    (6272, 184, 80, 0, 1),       # 14x14 projection with residual: ragged K (5.75 k-blocks), ragged N tile
    (1568, 960, 160, 0, 0),      # 7x7, deep K
    (100352, 16, 16, 0, 1),      # 112^2 x 8 images, K < one k-block
    (1000, 96, 576, 1, 0),       # M not a multiple of 128, wide N (cn layer)
])
def test_gemm_tc3x_matches_fp64(native_lib, M, K, N, relu, use_res):
    g = torch.Generator().manual_seed(61)
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    scale, bias = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    res = torch.randn(M, N, generator=g) if use_res else None
    ref = (a.double() @ w.double().t()) * scale.double() + bias.double()
    if res is not None:
        ref = ref + res.double()
    ref = (F.relu(ref) if relu else ref).float()
    hi, lo = tf32_split(w)
    d = [t.to(DEV) if t is not None else None for t in (a, hi, lo, scale, bias, res)]
    out = torch.full((M, N), float("nan"), device=DEV)
    rc = native_lib.smk_debug_gemm_tc3x(P(d[0]), K, M, P(d[1]), P(d[2]), P(d[3]), P(d[4]), N, K, relu, P(d[5]), N, P(out), N, stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    got = out.cpu()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    # the error left is the dropped a_lo*w_lo products and the tensor core's own accumulation, ~100x below plain TF32;
    # bound it at 4e-6 * sqrt(K / 64) of the output scale
    assert err <= 4e-6 * ref.abs().max().item() * max(1.0, (K / 64) ** 0.5), "max err %.3g vs scale %.3g" % (err, ref.abs().max().item())


@pytest.mark.parametrize("B,H,Cin,mid,stride", [(2, 28, 40, 120, 1), (1, 14, 80, 200, 1), (3, 56, 24, 72, 2), (1, 112, 16, 64, 2), (2, 14, 112, 672, 1),
                                                   (2, 20, 24, 72, 1), (3, 30, 16, 64, 2), (40, 28, 40, 120, 1)])
def test_xdw3x_matches_fp64(native_lib, B, H, Cin, mid, stride):
    g = torch.Generator().manual_seed(62)
    x = torch.randn(B, Cin, H, H, generator=g)
    w1 = torch.randn(mid, Cin, 1, 1, generator=g) / Cin ** 0.5
    s1, b1 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    wd = torch.randn(mid, 1, 3, 3, generator=g) / 3.0
    s2, b2 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    dd = torch.float64
    e = F.relu(F.conv2d(x.to(dd), w1.to(dd)) * s1.to(dd).view(1, -1, 1, 1) + b1.to(dd).view(1, -1, 1, 1))
    ref = F.relu(tf_same_dw(e, wd.to(dd), stride) * s2.to(dd).view(1, -1, 1, 1) + b2.to(dd).view(1, -1, 1, 1)).float()
    Ho = (H + stride - 1) // stride
    hi, lo = tf32_split(w1.view(mid, Cin))
    xd, wdd = nhwc(x).to(DEV), wd.view(mid, 9).t().contiguous().to(DEV)
    t = [hi.to(DEV), lo.to(DEV), s1.to(DEV), b1.to(DEV), s2.to(DEV), b2.to(DEV)]
    out = torch.full((B, Ho, Ho, mid), float("nan"), device=DEV)
    rc = native_lib.smk_debug_xdw3x(P(xd), B, H, H, Cin, P(t[0]), P(t[1]), P(t[2]), P(t[3]), mid, P(wdd), P(t[4]), P(t[5]), stride, P(out), stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu()
    assert torch.isfinite(got).all(), "unwritten outputs: %d" % int((~torch.isfinite(got)).sum())
    err = (got - ref).abs().max().item()
    assert err <= 5e-6 * ref.abs().max().item(), "max err %.3g vs scale %.3g" % (err, ref.abs().max().item())


# ----------------------------------------------------------------- persistent windowed 3x3 conv (conv3_win_tc.cu)
def run_win(native_lib, x, w, scale, bias, relu):
    B, Cin, H, W = x.shape
    N = w.shape[0]
    xd, wd = nhwc(x).to(DEV), w_nk(w).to(DEV)
    out = torch.full((B, H, W, N), float("nan"), device=DEV)
    sd, bd = scale.to(DEV), bias.to(DEV)
    rc = native_lib.smk_debug_conv3_win(P(xd), Cin, B, H, W, Cin, P(wd), P(sd), P(bd), N, relu, P(out), N, stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    return out.permute(0, 3, 1, 2).cpu()


def test_conv3_win_exact_on_small_integers(native_lib):
    """Operands exactly representable in TF32: the result must be exact — pins the patch addressing (tap views into the
    swizzled window, wrap columns, zero-filled halo), the resident-weight indexing, the tile decode and the split of the
    tiles over the two pipelines of a CTA."""
    g = torch.Generator().manual_seed(71)
    for (B, H, W, Cin, N) in [(2, 61, 70, 32, 32), (1, 56, 56, 64, 32), (3, 57, 113, 32, 64), (1, 60, 56, 32, 32),
                              (1, 60, 64, 64, 64), (2, 57, 59, 128, 64)]:          # the last two stream their weights through the ring
        x = torch.randint(-3, 4, (B, Cin, H, W), generator=g).float()
        w = torch.randint(-2, 3, (N, Cin, 3, 3), generator=g).float()
        one, zero = torch.ones(N), torch.zeros(N)
        ref = F.conv2d(x.double(), w.double(), padding=1).float()
        got = run_win(native_lib, x, w, one, zero, 0)
        assert torch.isfinite(got).all(), "unwritten outputs: %d" % int((~torch.isfinite(got)).sum())
        assert torch.equal(got, ref), "B %d H %d W %d Cin %d N %d: %d mismatches" % (B, H, W, Cin, N, int((got != ref).sum()))


@pytest.mark.parametrize("B,H,W,Cin,N", [(2, 224, 224, 32, 32), (1, 224, 224, 64, 32), (2, 112, 112, 32, 64), (5, 64, 90, 32, 32),
                                         (2, 112, 112, 64, 64), (1, 112, 112, 128, 64)])
def test_conv3_win_random_with_epilogue(native_lib, B, H, W, Cin, N):
    x, w, scale, bias = make_case(B, H, W, Cin, N, 72, 1)
    for relu in (1, 0):
        ref = torch_conv(x, w, scale, bias, 1, relu)
        got = run_win(native_lib, x, w, scale, bias, relu)
        assert torch.isfinite(got).all()
        assert (got - ref).abs().max().item() <= 3e-3 * ref.abs().max().item()
