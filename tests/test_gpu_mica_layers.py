"""MICA's convolutions one at a time against float64: every distinct layer shape the network issues, each with the epilogue
it uses, through the kernel-test entry points smk_debug_mica_conv / smk_debug_mica_gather_s2 (csrc/mica.cu), at B = 1 and 2
(7^2 * B rows are not a multiple of the 128-row tile) and precisions 0, 1 and 3.

- Small-integer data (inputs, weights, residuals and biases small integers, scales and PReLU slopes powers of two) makes
  every operand exact in TF32 and every sum exact in fp32: the outputs must equal float64 bit for bit.
- Random data must stay within a bound derived from K: |out - ref| <= (K + 16) 2^-22 S + 2^-11 |ref| [TF32-rounded
  outputs], where S is the sum of the magnitudes that enter the output (|scale| sum_k |a w| + |bias| + |res|), carried
  through the second store's affine.
"""
import ctypes as C
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (name, mode, H out, Cin, N, epilogue): mode 1 = 3x3 conv (K = 9 Cin), mode 0 = GEMM over a gathered matrix (K = Cin);
# epilogue "prelu" (stem: also the affine second store), "res2" (residual + affine second store), "res" (residual only),
# "plain"
LAYERS = [("stem", 1, 112, 32, 64, "prelu2"), ("stem_f32", 1, 112, 4, 64, "prelu2"),
          ("conv1_112_64_64", 1, 112, 64, 64, "prelu"), ("conv1_56_64_64", 1, 56, 64, 64, "prelu"),
          ("conv1_56_64_128", 1, 56, 64, 128, "prelu"), ("conv1_28_128_128", 1, 28, 128, 128, "prelu"),
          ("conv1_28_128_256", 1, 28, 128, 256, "prelu"), ("conv1_14_256_256", 1, 14, 256, 256, "prelu"),
          ("conv1_14_256_512", 1, 14, 256, 512, "prelu"), ("conv1_7_512_512", 1, 7, 512, 512, "prelu"),
          ("conv2_56", 1, 56, 64, 64, "res2"), ("conv2_28", 1, 28, 128, 128, "res2"), ("conv2_14", 1, 14, 256, 256, "res2"),
          ("conv2_7", 1, 7, 512, 512, "res2"), ("conv2_7_last", 1, 7, 512, 512, "res"),
          ("conv2_s2_56", 0, 56, 576, 64, "res2"), ("conv2_s2_28", 0, 28, 1152, 128, "res2"),
          ("conv2_s2_14", 0, 14, 2304, 256, "res2"), ("conv2_s2_7", 0, 7, 4608, 512, "res2"),
          ("ds_56", 0, 56, 64, 64, "plain"), ("ds_28", 0, 28, 64, 128, "plain"), ("ds_14", 0, 14, 128, 256, "plain"),
          ("ds_7", 0, 7, 256, 512, "plain"), ("fc", 0, 1, 25088, 512, "plain")]
GATHERS = [(112, 64, 9), (56, 128, 9), (28, 256, 9), (14, 512, 9), (112, 64, 1), (56, 64, 1), (28, 128, 1), (14, 256, 1)]

_vp, _i = C.c_void_p, C.c_int


@pytest.fixture(scope="module")
def L(native_lib):
    native_lib.smk_debug_mica_conv.restype = _i
    native_lib.smk_debug_mica_conv.argtypes = [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp,
                                               _vp, _i, _i, _vp, _i, _vp, _vp, _i, _vp]
    native_lib.smk_debug_mica_gather_s2.restype = _i
    native_lib.smk_debug_mica_gather_s2.argtypes = [_vp, _i, _i, _i, _i, _i, _vp, _vp]
    return native_lib


def rna(t):
    """fp32 -> TF32, round to nearest, ties away (cvt.rna.tf32.f32)."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def ptr(t):
    return None if t is None else t.data_ptr()


def _skip_unsupported(spec, precision):
    if spec[0] == "stem_f32" and precision != 0:
        pytest.skip("the fp32 stem's 4 padded input channels; the tensor-core stem reads 32")


def _data(spec, B, integer, precision, g):
    name, mode, H, Cin, N, epi = spec
    K = 9 * Cin if mode == 1 else Cin
    rows = B * H * H if name != "fc" else B
    if integer:
        ri = lambda *s: torch.randint(-2, 3, s, generator=g).float()                         # noqa: E731
        p2 = lambda n, lo, hi: 2.0 ** torch.randint(lo, hi, (n,), generator=g).float()    # noqa: E731
        x, w = ri(rows, Cin) if mode == 0 else ri(B, H, H, Cin), ri(N, K)
        scale, bias, res = p2(N, -1, 2), ri(N), ri(rows, N)
        prelu, scale2, bias2 = p2(N, -2, 0), p2(N, -1, 2), ri(N)
    else:
        x = torch.randn(rows, Cin, generator=g) if mode == 0 else torch.randn(B, H, H, Cin, generator=g)
        w = torch.randn(N, K, generator=g) * (2.0 / K) ** 0.5
        scale, bias, res = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1, torch.randn(rows, N, generator=g)
        prelu, scale2, bias2 = torch.rand(N, generator=g) * 0.5, torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    if precision == 1:
        x = rna(x)                                   # the layer's input is a TF32-rounded activation at precision 1
    d = dict(x=x, w=w, scale=scale, bias=bias, res=res if epi.startswith("res") else None,
             prelu=prelu if epi.startswith("prelu") else None)
    if epi in ("prelu2", "res2"):
        d.update(scale2=scale2, bias2=bias2)
    return d


def _oracle(spec, d, B, w_used):
    """float64 (out, out2, S): S bounds the magnitudes that enter each output."""
    name, mode, H, Cin, N, epi = spec
    x, w = d["x"].double(), w_used.double()
    if mode == 1:
        wc = w.view(N, 3, 3, Cin).permute(0, 3, 1, 2)
        xc = x.permute(0, 3, 1, 2)
        acc = F.conv2d(xc, wc, padding=1).permute(0, 2, 3, 1).reshape(-1, N)
        mag = F.conv2d(xc.abs(), wc.abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    else:
        acc, mag = x @ w.t(), x.abs() @ w.abs().t()
    v = acc * d["scale"].double() + d["bias"].double()
    S = mag * d["scale"].double().abs() + d["bias"].double().abs()
    if d["res"] is not None:
        v = v + d["res"].double()
        S = S + d["res"].double().abs()
    if d["prelu"] is not None:
        v = torch.where(v < 0, v * d["prelu"].double(), v)
    v2 = S2 = None
    if "scale2" in d:
        v2 = v * d["scale2"].double() + d["bias2"].double()
        S2 = S * d["scale2"].double().abs() + d["bias2"].double().abs()
    return v, v2, S, S2


def _run(L, spec, d, B, precision):
    name, mode, H, Cin, N, epi = spec
    K = 9 * Cin if mode == 1 else Cin
    rows = B * H * H if name != "fc" else B
    w = d["w"]
    w_kn = wt_hi = wt_lo = None
    if precision == 0:
        w_kn, w_used = w.t().contiguous().to(DEV), w
    else:
        hi = rna(w)
        wt_hi, w_used = hi.to(DEV), hi
        if precision == 3:
            wt_lo, w_used = rna(w - hi).to(DEV), w
    dv = {k: (v.to(DEV).contiguous() if v is not None else None) for k, v in d.items()}
    out = torch.full((rows, N), float("nan"), device=DEV)
    out2 = torch.full((rows, N), float("nan"), device=DEV) if "scale2" in d else None
    rnd = 1 if precision == 1 else 0
    round_out = rnd if epi.startswith("prelu") or name == "conv2_7_last" else 0
    bh, bw = (1, B) if name == "fc" else (H, H)
    rc = L.smk_debug_mica_conv(ptr(dv["x"]), Cin, B if name != "fc" else 1, bh, bw, Cin, ptr(w_kn), ptr(wt_hi), ptr(wt_lo),
                               ptr(dv["scale"]), ptr(dv["bias"]), N, K, mode, ptr(dv["res"]), N, ptr(dv["prelu"]), ptr(out), N,
                               round_out, ptr(out2), N, ptr(dv.get("scale2")), ptr(dv.get("bias2")), rnd, None)
    assert rc == 0, L.smk_last_error()
    torch.cuda.synchronize()
    return out.cpu(), (out2.cpu() if out2 is not None else None), w_used, bool(round_out), bool(rnd)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("spec", LAYERS, ids=[s[0] for s in LAYERS])
def test_layer_integer_data_is_exact(L, spec, precision, B):
    _skip_unsupported(spec, precision)
    g = torch.Generator().manual_seed(zlib.crc32(("%s %d" % (spec[0], B)).encode()))
    d = _data(spec, B, True, precision, g)
    out, out2, w_used, r1, r2 = _run(L, spec, d, B, precision)
    v, v2, _, _ = _oracle(spec, d, B, w_used)
    exact = lambda t, r: rna(t.float()) if r else t.float()                 # noqa: E731  (TF32-rounded stores)
    assert torch.equal(out, exact(v, r1)), spec[0]
    if v2 is not None:
        assert torch.equal(out2, exact(v2, r2)), spec[0]


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("spec", LAYERS, ids=[s[0] for s in LAYERS])
def test_layer_random_data_within_k_bound(L, spec, precision, B):
    _skip_unsupported(spec, precision)
    g = torch.Generator().manual_seed(7 + zlib.crc32(("%s %d" % (spec[0], B)).encode()))
    d = _data(spec, B, False, precision, g)
    out, out2, w_used, r1, r2 = _run(L, spec, d, B, precision)
    v, v2, S, S2 = _oracle(spec, d, B, w_used)
    K = 9 * spec[3] if spec[1] == 1 else spec[3]
    eps = (K + 16) * 2.0 ** -22
    worst = 0.0
    for got, ref, mag, rounded in ((out, v, S, r1), (out2, v2, S2, r2)):
        if got is None:
            continue
        bound = eps * mag + (2.0 ** -11 * ref.abs() if rounded else 0.0) + 1e-30
        ratio = ((got.double() - ref).abs() / bound).max().item()
        worst = max(worst, ratio)
    print("%s B=%d precision %d: err / bound %.3f" % (spec[0], B, precision, worst))
    assert worst <= 1.0


@pytest.mark.parametrize("round_", [0, 1])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("H,C,taps", GATHERS)
def test_gather_s2(L, H, C, taps, B, round_):
    g = torch.Generator().manual_seed(H * 7 + C + taps + B)
    x = torch.randn(B, H, H, C, generator=g)
    Ho = H // 2
    out = torch.full((B * Ho * Ho, taps * C), float("nan"), device=DEV)
    xd = x.to(DEV)
    assert L.smk_debug_mica_gather_s2(xd.data_ptr(), B, H, C, taps, round_, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    xc = x.permute(0, 3, 1, 2)
    if taps == 9:
        u = F.unfold(xc, 3, padding=1, stride=2)                            # [B, C*9, Ho*Ho], index c*9 + tap
        want = u.view(B, C, 9, Ho * Ho).permute(0, 3, 2, 1).reshape(B * Ho * Ho, 9 * C)
    else:
        want = xc[:, :, ::2, ::2].permute(0, 2, 3, 1).reshape(B * Ho * Ho, C)
    if round_:
        want = rna(want)
    assert torch.equal(out.cpu(), want)
