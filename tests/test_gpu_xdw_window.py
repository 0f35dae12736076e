"""GPU suite (-m gpu): the fused expand 1x1 + depthwise 3x3 kernel (xdw_tc.cu) on every encoder layer shape of
tools/bench_xdw.py, through both entry points (plain TF32 and 3xTF32).  On small integers every product and sum is
exact in TF32 and fp32, so the kernel must equal the CPU result bit for bit whatever its k-step count, window
buffering or tile edges; on random data it is held to the fp64 reference at the tolerances of test_gpu_kernels.py."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tools.bench_xdw import SHAPES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B = 2
LAYERS = sorted({(H, Cin, mid, stride) for (H, Cin, mid, stride, _) in SHAPES})


def P(t):
    return C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def tf_same_dw(e, wdw, stride):
    """Depthwise 3x3 with TF-'SAME' padding: symmetric for stride 1, bottom/right for stride 2."""
    if stride == 1:
        return F.conv2d(e, wdw, padding=1, groups=e.shape[1])
    return F.conv2d(F.pad(e, (0, 1, 0, 1)), wdw, stride=2, groups=e.shape[1])


def reference(x, w1, s1, b1, wd, s2, b2, stride):
    dd = torch.float64
    bn = lambda t, s, b: t * s.to(dd).view(1, -1, 1, 1) + b.to(dd).view(1, -1, 1, 1)
    e = F.relu(bn(F.conv2d(x.to(dd), w1.to(dd)), s1, b1))
    return F.relu(bn(tf_same_dw(e, wd.to(dd), stride), s2, b2)).float()


def tf32_split(w):
    """hi = tf32(w) (round to nearest, ties away), lo = tf32(w - hi): the encoder's packing of the 3xTF32 weights."""
    rna = lambda t: ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    hi = rna(w)
    return hi, rna(w - hi)


def run(native_lib, x3, x, w1, s1, b1, wd, s2, b2, stride):
    Bx, Cin, H, _ = x.shape
    mid = w1.shape[0]
    Ho = (H + stride - 1) // stride
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    wdd = wd.view(mid, 9).t().contiguous().to(DEV)
    s1d, b1d, s2d, b2d = s1.to(DEV), b1.to(DEV), s2.to(DEV), b2.to(DEV)
    out = torch.full((Bx, Ho, Ho, mid), float("nan"), device=DEV)
    if x3:
        hi, lo = [t.to(DEV) for t in tf32_split(w1.view(mid, Cin))]
        rc = native_lib.smk_debug_xdw3x(P(xd), Bx, H, H, Cin, P(hi), P(lo), P(s1d), P(b1d), mid, P(wdd), P(s2d), P(b2d), stride,
                                        P(out), stream())
    else:
        w1d = w1.view(mid, Cin).contiguous().to(DEV)
        rc = native_lib.smk_debug_xdw(P(xd), Bx, H, H, Cin, P(w1d), P(s1d), P(b1d), mid, P(wdd), P(s2d), P(b2d), stride, 0, P(out),
                                      stream())
    assert rc == 0, native_lib.smk_last_error()
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu()
    assert torch.isfinite(got).all(), "unwritten outputs: %d" % int((~torch.isfinite(got)).sum())
    return got


def test_layer_shapes_cover_edges():
    # output tiles are 14x14 (stride 1) or 7x7 (stride 2): at least one layer has a partial edge tile, and at least
    # one has a last channel chunk narrower than 32
    assert any(((H + s - 1) // s) % (14 if s == 1 else 7) for (H, _, _, s) in LAYERS)
    assert any(mid % 32 for (_, _, mid, _) in LAYERS)


@pytest.mark.parametrize("x3", [0, 1], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("H,Cin,mid,stride", LAYERS)
def test_xdw_exact_on_small_integers(native_lib, H, Cin, mid, stride, x3):
    g = torch.Generator().manual_seed(1000 * H + Cin + mid + stride)
    x = torch.randint(-2, 3, (B, Cin, H, H), generator=g).float()
    w1 = torch.randint(-1, 2, (mid, Cin, 1, 1), generator=g).float()
    wd = torch.randint(-1, 2, (mid, 1, 3, 3), generator=g).float()
    one, zero = torch.ones(mid), torch.zeros(mid)
    ref = F.relu(tf_same_dw(F.relu(F.conv2d(x.double(), w1.double())), wd.double(), stride)).float()
    got = run(native_lib, x3, x, w1, one, zero, wd, one, zero, stride)
    assert torch.equal(got, ref), "%d of %d outputs differ" % (int((got != ref).sum()), ref.numel())


@pytest.mark.parametrize("x3", [0, 1], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("H,Cin,mid,stride", LAYERS)
def test_xdw_matches_fp64(native_lib, H, Cin, mid, stride, x3):
    g = torch.Generator().manual_seed(2000 * H + Cin + mid + stride)
    x = torch.randn(B, Cin, H, H, generator=g)
    w1 = torch.randn(mid, Cin, 1, 1, generator=g) / Cin ** 0.5
    s1, b1 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    wd = torch.randn(mid, 1, 3, 3, generator=g) / 3.0
    s2, b2 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    ref = reference(x, w1, s1, b1, wd, s2, b2, stride)
    got = run(native_lib, x3, x, w1, s1, b1, wd, s2, b2, stride)
    err = (got - ref).abs().max().item()
    tol = 5e-6 if x3 else 3e-3
    assert err <= tol * ref.abs().max().item(), "max err %.3g vs scale %.3g" % (err, ref.abs().max().item())
