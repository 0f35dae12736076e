"""GPU suite (-m gpu) for the generator's 3xTF32 precision (SmirkGenerator.precision = 3).

Kernel checks go through smk_debug_conv_tc3x, one tensor-core convolution at a time, at every layer shape the
(6, 3, 32, 5) generator issues in its forward and its input gradient, with the epilogue options that layer uses, at B = 1
and 2.  Small-integer operands are exact in TF32 (tails zero) and every sum stays below 2^24, so the result must equal
float64 bit for bit.  On random data the bound is derived below from K and 2^-22.

Module checks run the precision-3 generator against the fp32 oracles at 1e-4 of the max-abs, and pin its determinism,
batch independence, launch count, CUDA-graph capture and the full-cycle pipeline."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from smirk_b200 import synth_inputs

from test_gpu_generator_grad import device_grad, gen, inputs, replay_grad
from test_gpu_kernels import P, nhwc, stream, tf32_split, w_nk
from test_gpu_parity import rel_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -22

# ----------------------------------------------------------------------------------------------------- error bound
# With a = a_hi + a_lo and w = w_hi + w_lo (hi = tf32 round-to-nearest, so |a_lo| <= 2^-11 |a|, |w_lo| <= 2^-11 |w|), one
# 3xTF32 product a_hi w_hi + a_lo w_hi + a_hi w_lo differs from a w by
#   the dropped a_lo w_lo             <= 2^-22 |a w|,
#   a_lo truncated to TF32 by wgmma   <= 2^-10 |a_lo| |w| <= 2^-21 |a w|,
#   w_lo rounded to TF32 on the host  <= 2^-11 |w_lo| |a| <= 2^-22 |a w|,
# so <= 4 * 2^-22 |a w|, and with independent signs over the K products their sum stays within a few times
# 4 * 2^-22 ||a w||_2 (the L2 norm over k of one output's products).  The accumulator takes 3 K / 8 wgmma updates (three per
# 8-deep k-step), each truncating up to 2^-23 of a partial sum that grows like a random walk to ||a w||_2; truncation keeps
# losing magnitude in the same direction, so these add up to about 2^-22 (K / 8) ||a w||_2 (measured: 1.7x a sqrt(K) bound
# at K = 288).  The generator's kernel (X3 = 3) sums each 32-deep k-block apart and adds it in fp32, which removes most of
# that; the bound still allows it, with a 2x margin: 2^-22 (8 + K / 4) ||a w||_2, times |scale|, plus 2^-22 of the
# epilogue's operands (the fp32 fma and residual add).  Plain TF32 (per-product error ~2^-11 |a w|) misses it by 25x at
# K = 288; at K = 4608 the margin shrinks below 2x, and the small-integer checks, exact at every K, pin the arithmetic there.
def bound(K, norm, scale, acc, bias, res=None):
    b = EPS * ((8 + K / 4) * norm * scale.abs() + (acc * scale).abs() + bias.abs())
    return b + EPS * res.abs() if res is not None else b


def head_bound(z, act, act_bnd, hw, hb):
    """Head output sigmoid(hb + act . hw): the activations' error through |hw| and the 32-term fp32 sum, then
    sigmoid' <= 1/4 and __expf's relative error (2 + 1.16 |z|) ulp, plus the final division."""
    dz = act_bnd @ hw.abs() + 64 * EPS * (act.abs() @ hw.abs() + hb.abs())
    return 0.25 * (dz + 4 * EPS * (2 + 1.2 * z.abs())) + EPS


# ---------------------------------------------------------------------------------------------------- one call
def conv_tc3x(L):
    """smk_debug_conv_tc3x with its argument types: a kernel-test entry point of gemm_tc.cu that is exported but not
    declared in include/smirk_b200.h, so _lib.BINDINGS does not set them."""
    fn = L.smk_debug_conv_tc3x
    vp, i = C.c_void_p, C.c_int
    fn.restype = i
    fn.argtypes = [vp, i, i, i, i, i, vp, vp, vp, vp, i, i, i, i, vp, i, i, vp, i, i, vp, i, vp, i, vp, vp, i, vp]
    return fn


def conv3x(L, x, w, scale, bias, mode, relu, res=None, res_pad=0, store=0, ld_out=None, mask=None, out2=False, head=None):
    """x [B,Cin,H,W], w [N,Cin,k,k] (k = 1 for mode 0), all float32 on the host -> (out, out2) as the kernel wrote them.
    res [B,N,H,W] (res_pad: read from the interior of a padded buffer), mask [B,H,W,N] NHWC, head = (hw [N][hc], hb [hc])."""
    B, Cin, H, W = x.shape
    N = w.shape[0]
    xd = nhwc(x).to(DEV)
    if mode == 2:
        buf = torch.zeros(B, H + 2, W + 2, Cin, device=DEV)
        buf[:, 1:-1, 1:-1] = xd
        assert L.smk_debug_reflect_halo(P(buf), B, H, W, Cin, stream()) == 0
        xd = buf
    hi, lo = (t.to(DEV) for t in tf32_split(w_nk(w)))
    K = hi.shape[1]
    ld_out = ld_out or N
    shape = {0: (B, H, W, ld_out), 1: (B, 2 * H, 2 * W, ld_out), 2: (B, H + 2, W + 2, ld_out)}.get(store)
    out = torch.full(shape if store != 3 else (B, head[0].shape[1], H, W), float("nan"), device=DEV)
    resd = None
    if res is not None:
        resd = nhwc(res).to(DEV)
        if res_pad:
            resd = F.pad(resd, (0, 0, 1, 1, 1, 1)).contiguous()
    maskd = mask.to(DEV) if mask is not None else None
    o2 = torch.full((B, H, W, N), float("nan"), device=DEV) if out2 else None
    hw, hb = (head[0].to(DEV), head[1].to(DEV)) if head else (None, None)
    sd, bd = scale.to(DEV), bias.to(DEV)
    rc = conv_tc3x(L)(P(xd), Cin, B, H, W, Cin, P(hi), P(lo), P(sd), P(bd), N, K, mode, relu, P(resd), N, res_pad,
                      P(out), ld_out, store, P(maskd), N, P(o2), N, P(hw), P(hb), head[0].shape[1] if head else 0, stream())
    assert rc == 0, L.smk_last_error()
    torch.cuda.synchronize()
    return out.cpu(), (o2.cpu() if out2 else None)


def reference(x, w, mode):
    """-> (acc, norm) NHWC float64: the convolution without epilogue and the L2 norm over k of each output's products."""
    x, w = x.double(), w.double()
    pad = (lambda t: F.pad(t, (1, 1, 1, 1), mode="reflect")) if mode == 2 else (lambda t: t)
    p = 1 if mode == 1 else 0
    acc = F.conv2d(pad(x), w, padding=p)
    norm = F.conv2d(pad(x * x), w * w, padding=p).sqrt()
    return acc.permute(0, 2, 3, 1), norm.permute(0, 2, 3, 1)


def operands(B, S, Cin, N, k, seed, ints):
    g = torch.Generator().manual_seed(seed)
    if ints:
        return (torch.randint(-3, 4, (B, Cin, S, S), generator=g).float(), torch.randint(-2, 3, (N, Cin, k, k), generator=g).float(),
                torch.randint(1, 3, (N,), generator=g).float(), torch.randint(-2, 3, (N,), generator=g).float())
    return (torch.randn(B, Cin, S, S, generator=g), torch.randn(N, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5,
            torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1)


def compare(got, ref, bnd, ints, what):
    assert torch.isfinite(got).all(), "%s: %d unwritten / non-finite outputs" % (what, int((~torch.isfinite(got)).sum()))
    if ints:
        assert torch.equal(got, ref.float()), "%s: %d of %d differ from float64" % (what, int((got != ref.float()).sum()), got.numel())
    else:
        err = (got.double() - ref).abs()
        assert bool((err <= bnd).all()), "%s: %d outside the bound, worst err / bound %.3g" % (what, int((err > bnd).sum()), float((err / bnd).max()))


# --------------------------------------------------------------------------------- 3x3 layers: (S, Cin, N) of the
# forward convolutions (Cin -> N) and of the dgrads (cout -> cin), zero padding; the first layer's 6 inputs are padded to 32
ZERO_PAD = [(224, 32, 32), (224, 64, 32), (224, 32, 64), (112, 32, 64), (112, 64, 64), (112, 64, 32), (112, 128, 64), (112, 64, 128),
            (56, 64, 128), (56, 128, 128), (56, 128, 64), (56, 256, 128), (56, 128, 256), (28, 128, 256), (28, 256, 256),
            (28, 256, 128), (28, 512, 256), (28, 256, 512), (14, 256, 512), (14, 512, 512), (14, 512, 256), (16, 512, 512)]


@pytest.mark.parametrize("B", (1, 2))
@pytest.mark.parametrize("S,Cin,N", ZERO_PAD)
@pytest.mark.parametrize("ints", (True, False), ids=("ints", "random"))
def test_conv3x3_layer(native_lib, S, Cin, N, B, ints):
    """The forward's form (ReLU, a channel slice of a concat buffer, the second compact store) and the dgrad's form
    (no ReLU, the saved activation's mask)."""
    x, w, s, b = operands(B, S, Cin, N, 3, S + Cin + N + B, ints)
    acc, norm = reference(x, w, 1)
    y = acc * s.double() + b.double()
    bnd = bound(9 * Cin, norm, s.double(), acc, b.double())
    out, o2 = conv3x(native_lib, x, w, s, b, 1, 1, ld_out=2 * N, out2=True)
    compare(out[..., :N], y.clamp_min(0), bnd, ints, "relu")
    assert torch.isnan(out[..., N:]).all()
    compare(o2, y.clamp_min(0), bnd, ints, "out2")
    g = torch.Generator().manual_seed(S * N)
    mask = torch.randint(-1, 2, (B, S, S, N), generator=g).float()
    out, _ = conv3x(native_lib, x, w, s, b, 1, 0, mask=mask)
    compare(out, torch.where(mask > 0, y, 0.0), bnd, ints, "mask")


@pytest.mark.parametrize("B", (1, 2))
@pytest.mark.parametrize("ints", (True, False), ids=("ints", "random"))
def test_resnet_conv_reflection_padded(native_lib, B, ints):
    """The ResNet block convs (14^2, 512 -> 512, mode 2): conv1 with ReLU into the interior of a padded buffer plus the
    compact copy; conv2 without ReLU, the residual read from a padded buffer, stored padded and plain."""
    S, C = 14, 512
    x, w, s, b = operands(B, S, C, C, 3, 40 + B, ints)
    acc, norm = reference(x, w, 2)
    y = acc * s.double() + b.double()
    bnd = bound(9 * C, norm, s.double(), acc, b.double())
    out, o2 = conv3x(native_lib, x, w, s, b, 2, 1, store=2, out2=True)
    compare(out[:, 1:-1, 1:-1], y.clamp_min(0), bnd, ints, "store 2")
    assert torch.isnan(out[:, 0]).all() and torch.isnan(out[:, :, 0]).all() and torch.isnan(out[:, -1]).all()
    compare(o2, y.clamp_min(0), bnd, ints, "out2")
    g = torch.Generator().manual_seed(41 + B)
    res = torch.randint(-3, 4, (B, C, S, S), generator=g).float() if ints else torch.randn(B, C, S, S, generator=g)
    r = nhwc(res).double()
    bnd_r = bound(9 * C, norm, s.double(), acc, b.double(), r)
    for store in (2, 0):
        out, _ = conv3x(native_lib, x, w, s, b, 2, 0, res=res, res_pad=1, store=store)
        compare(out[:, 1:-1, 1:-1] if store == 2 else out, y + r, bnd_r, ints, "residual, store %d" % store)
    out, _ = conv3x(native_lib, x, w, s, b, 2, 1, res=res, res_pad=0)             # plain residual + ReLU
    compare(out, (y + r).clamp_min(0), bnd_r, ints, "plain residual")


# (S, Cin, Cout) of the four transposed convolutions: one GEMM with N = 4 Cout, pixel-shuffled into the lower half of a
# concat buffer; and their dgrads: a GEMM with K = 4 Cout, N = Cin, masked
UPCONV = [(14, 512, 256), (28, 256, 128), (56, 128, 64), (112, 64, 32)]


@pytest.mark.parametrize("B", (1, 2))
@pytest.mark.parametrize("S,Cin,Cout", UPCONV)
@pytest.mark.parametrize("ints", (True, False), ids=("ints", "random"))
def test_upconv_and_its_dgrad(native_lib, S, Cin, Cout, B, ints):
    x, w, _, bias = operands(B, S, Cin, 4 * Cout, 1, S + Cin + B, ints)
    one = torch.ones(4 * Cout)
    acc, norm = reference(x, w, 0)
    y = acc + bias.double()
    bnd = bound(Cin, norm, one.double(), acc, bias.double())
    out, _ = conv3x(native_lib, x, w, one, bias, 0, 0, store=1, ld_out=2 * Cout)
    shuf = lambda t: t.reshape(B, S, S, 2, 2, Cout).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * S, 2 * S, Cout)
    compare(out[..., :Cout], shuf(y), shuf(bnd), ints, "store 1")
    assert torch.isnan(out[..., Cout:]).all()
    g, _, s, b = operands(B, S, 4 * Cout, Cin, 1, 7 * S + B, ints)
    wd = operands(B, S, 4 * Cout, Cin, 1, 9 * S + B, ints)[1]
    acc, norm = reference(g, wd, 0)
    y = acc * s.double() + b.double()
    mask = torch.randint(-1, 2, (B, S, S, Cin), generator=torch.Generator().manual_seed(S)).float()
    out, _ = conv3x(native_lib, g, wd, s, b, 0, 0, mask=mask)
    compare(out, torch.where(mask > 0, y, 0.0), bound(4 * Cout, norm, s.double(), acc, b.double()), ints, "dgrad")


@pytest.mark.parametrize("B", (1, 2))
@pytest.mark.parametrize("ints", (True, False), ids=("ints", "random"))
def test_fused_head(native_lib, B, ints):
    """dec1conv2 + the 1x1 head + sigmoid (store 3, N = 32, three head channels), with and without the compact copy of
    the activations; 224^2 x B pixels, and a 9 x 11 image whose 99 pixels are less than one 128-row tile."""
    for S in (224, (9, 11)):
        Hh, Ww = (S, S) if isinstance(S, int) else S
        g = torch.Generator().manual_seed(50 + B)
        _, w, s, b = operands(B, 1, 32, 32, 3, 60 + B, ints)
        x = (torch.randint(-3, 4, (B, 32, Hh, Ww), generator=g).float() if ints else torch.randn(B, 32, Hh, Ww, generator=g))
        hw = (torch.randint(-1, 2, (32, 3), generator=g).float() * 0.25) if ints else torch.randn(32, 3, generator=g) * 0.2
        hb = torch.randn(3, generator=g) * 0.1
        acc, norm = reference(x, w, 1)
        act = (acc * s.double() + b.double()).clamp_min(0)
        bnd = bound(288, norm, s.double(), acc, b.double())
        z = act @ hw.double() + hb.double()
        want = torch.sigmoid(z).permute(0, 3, 1, 2)
        hbnd = head_bound(z, act, torch.zeros_like(bnd) if ints else bnd, hw.double(), hb.double()).permute(0, 3, 1, 2)
        for out2 in (False, True):
            out, o2 = conv3x(native_lib, x, w, s, b, 1, 1, store=3, out2=out2, head=(hw, hb))
            assert torch.isfinite(out).all()
            err = (out.double() - want).abs()
            assert bool((err <= hbnd).all()), "head: worst err / bound %.3g" % float((err / hbnd).max())
            if out2:
                compare(o2, act, bnd, ints, "head out2")


# ------------------------------------------------------------------------------------------------------ the module
FWD_CASES = [((6, 3, 32, 5), B) for B in (1, 2, 5)] + [((6, 3, 32, 0), 2), ((3, 1, 32, 1), 2)]


@pytest.mark.parametrize("cfg,B", FWD_CASES)
def test_forward_vs_oracle(native_lib, cfg, B):
    from oracle import generator_ref
    g = gen(cfg, 3)
    x, _ = inputs(cfg, B, 1300 + B + cfg[3])
    y = g(x.to(DEV))
    ref = generator_ref.generator_forward_ref({k: v.cpu() for k, v in g.state_dict().items()}, x, res_blocks=cfg[3])
    err = rel_close(y, ref, 1e-4)
    print("cfg %s B %d: forward max-abs err / max-abs %.2e" % (cfg, B, err / float(ref.abs().max())))


@pytest.mark.parametrize("cfg,B", FWD_CASES)
def test_input_grad_vs_replay_oracle(native_lib, cfg, B):
    g = gen(cfg, 3)
    x, gy = inputs(cfg, B, 1400 + B + cfg[3])
    got, _ = device_grad(g, x, gy)
    assert torch.isfinite(got).all()
    err = rel_close(got, replay_grad(g, x, gy), 1e-4)
    print("cfg %s B %d: input-gradient max-abs err / max-abs %.2e" % (cfg, B, err / float(got.abs().max())))


def test_against_plain_autograd(native_lib):
    """Reported, not gated: mask flips against the oracle's own fp32 forward, relative L2 error and cosine similarity
    of the input gradient against plain oracle autograd, for precisions 0, 1 and 3; asserted: cosine >= 0.99."""
    from oracle import generator_replay_ref as rr, make_golden_generator_grad as mg
    x, gy = mg.generator_input(), mg.upstream()
    xl = x.clone().requires_grad_()
    y, rec = rr.generator_activations_ref({k: v.cpu() for k, v in gen().state_dict().items()}, xl)
    ref = torch.autograd.grad((y * gy).sum(), xl)[0].double()
    rec = {k: v.detach() for k, v in rec.items()}
    for precision in (0, 1, 3):
        g = gen(precision=precision)
        got = device_grad(g, x, gy)[0].cpu().double()
        sv = g.saved_activations(x.to(DEV))
        flips = sum(int(((sv[k].cpu() > 0) != (rec[k] > 0)).sum()) for k in rec)
        rl2 = float((got - ref).norm() / ref.norm())
        cos = float((got * ref).sum() / (got.norm() * ref.norm()))
        print("precision %d: %d mask flips of %d, rel L2 %.2e, cosine %.6f"
              % (precision, flips, sum(v.numel() for v in rec.values()), rl2, cos))
        assert cos >= 0.99


def test_init_features_16_and_precision_2_raise(native_lib):
    """init_features = 16 is refused on the tensor cores at precision 3 as at precision 1; precision 2 is no generator
    precision."""
    import smirk_b200
    for cfg, precision, match in (((3, 1, 16, 3), 1, "init_features"), ((3, 1, 16, 3), 3, "init_features"),
                                  ((6, 3, 32, 5), 2, "0, 1 or 3")):
        g = smirk_b200.SmirkGenerator(*cfg).eval().to(DEV)
        g.precision = precision
        with pytest.raises(RuntimeError, match=match):
            g(torch.zeros(1, cfg[0], 224, 224, device=DEV))


def test_deterministic_batch_independent_and_launch_count(native_lib):
    from smirk_b200 import _lib
    L = _lib.lib()
    g = gen(precision=3)
    x, gy = inputs(g._cfg, 4, 1600)
    xd = x.to(DEV)
    assert torch.equal(g(xd), g(xd))
    assert torch.equal(device_grad(g, x, gy)[0], device_grad(g, x, gy)[0])
    x, gy = inputs(g._cfg, 16, 1601)
    gf, yf = device_grad(g, x, gy)
    gs, ys = device_grad(g, x[9:12].contiguous(), gy[9:12].contiguous())
    assert torch.equal(gf[9:12], gs) and torch.equal(yf[9:12], ys)
    counts = {}
    for precision in (1, 3):
        h = gen(precision=precision)
        xl = x[:2].to(DEV).requires_grad_()
        h(xl)                                                          # handles and workspaces exist before counting
        n0 = L.smk_launch_count()
        with torch.no_grad():
            h(xl)
        n1 = L.smk_launch_count()
        y = h(xl)
        n2 = L.smk_launch_count()
        torch.autograd.grad(y, xl, gy[:2].to(DEV))
        n3 = L.smk_launch_count()
        counts[precision] = (n1 - n0, n2 - n1, n3 - n2)
    assert counts[3] == counts[1], counts


def test_cuda_graph_forward_backward(native_lib):
    g = gen(precision=3)
    x, gy = inputs(g._cfg, 2, 1700)
    sx, sgy = x.to(DEV).requires_grad_(), gy.to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            torch.autograd.grad((g(sx) * sgy).sum(), sx)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = g(sx)
        gx = torch.autograd.grad((y * sgy).sum(), sx)[0]
    x2, gy2 = inputs(g._cfg, 2, 1701)
    with torch.no_grad():
        sx.copy_(x2.to(DEV))
        sgy.copy_(gy2.to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    want, ye = device_grad(g, x2, gy2)
    assert torch.equal(gx, want) and torch.equal(y.detach(), ye.detach())


def test_pipeline_with_masking_stage(asset_root, native_lib):
    """The full cycle with a precision-3 generator and the device masking step, replayed from its CUDA graph: the
    generator's output equals an eager run of the same generator on the replay's own inputs."""
    import smirk_b200
    from smirk_b200.masking import MaskingStage
    from smirk_b200.pipeline import SmirkPipeline
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    enc = enc.eval().to(DEV)
    enc.precision = 3
    fl, rd = smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV)
    g = copy.deepcopy(gen(precision=3))
    st = MaskingStage(fl.faces_tensor, synth_inputs.face_probabilities(fl.faces_tensor.shape[0]), seed=5)
    pipe = SmirkPipeline(enc, fl, rd, g, device=DEV, slots=1, masking=st)
    img, hull = synth_inputs.images(3, 1800).to(DEV), synth_inputs.hull_masks(3, 1801).to(DEV)
    for _ in range(2):
        a = {k: v.clone() for k, v in pipe.replay(img, hull).items()}
        with torch.no_grad():
            y = g(torch.cat([a["rendered_img"], a["masked_img"]], 1))
        assert torch.equal(a["reconstructed_img"], y)
