"""GPU suite (-m gpu): the train-mode encoder kernels (smirk_b200/csrc/encoder_train.cu) one at a time, through the
smk_debug_train_* entry points (each runs the host helper of the train path), against plain torch in float64; then a
per-layer audit of one real train forward.

Two kinds of check per kernel:
* Small integers.  Inputs in {-2..2}: every product and partial sum is an integer of magnitude below 2^24 (a weight
  gradient over M <= 6e5 pixels sums to at most 4 M < 2.4e6), exact in fp32 and fp64 in any order, so the kernel must
  equal the reference bit for bit.  BatchNorm: the fp64 sums are exact, so mean = float(sum / M) bitwise; invstd is
  1 / sqrt rounded to fp64 and then to fp32, so it may sit 1 ulp from the correctly rounded value.
* Random fp32 data against fp64, with the bound derived at each check.  u = 2^-24 is the unit roundoff of fp32.

Shapes: every layer shape of both backbones (read from a train handle's saved layout) at B = 1 and 32, and forced edges
where the chunking of the reductions changes.  Every chunked kernel is also launched twice and must repeat bitwise."""
import ctypes as C

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from smirk_b200 import synth_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
MAX_CHUNKS, WGRAD_PART = 512, 1 << 22          # encoder_train.cu: kMaxChunks, kWgradPart


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def cdiv(a, b):
    return -(-a // b)


def f32(x):
    return torch.tensor(x, dtype=torch.float32).item()


def ints(shape, seed, lo=-2, hi=2):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float()


def randn(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV)


def ulp(x):
    """Spacing of fp32 at |x| (x: float32 tensor), as float64."""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def same(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.fixture(scope="module")
def L(native_lib):
    return native_lib


@pytest.fixture(scope="module")
def ws(L):
    """Scratch of the entry points: BN partials (512 * C * 16 bytes, C <= 1280) or 4M floats of split-K partials."""
    return torch.empty(24 << 20, dtype=torch.uint8, device=DEV)


@pytest.fixture(scope="module")
def topo(L):
    """The layers of the pose (small) and shape (large) backbones from a train handle's saved layout (the expression
    backbone is the shape one's): [(kind, H_in, C_in, H_out, C_out)], kind 'stem', 'dw' or 'pw', in layout order; and
    the heads' (feat, n_out)."""
    from smirk_b200 import _lib
    h = C.c_void_p()
    _lib.call("smk_encoder_train_create", DEV, 3, 300, 50, 0, C.byref(h))
    h = _lib.NativeHandle(h, "smk_encoder_destroy")
    n = _lib.call("smk_encoder_saved_bytes", DEV, h, 1) // 4
    views = _lib.saved_views("encoder", h, torch.empty(n), 1)
    layers, heads, act, feat = [], [], None, None
    for name, v in views.items():
        leaf = name.rsplit(".", 1)[1]
        if v.dim() == 2:                       # pooled [B, feat], then the head [B, n_out]
            if name.endswith(".pooled"):
                feat = v.shape[1]
            else:
                heads.append((feat, v.shape[1]))
            continue
        _, c, hh, _ = v.shape
        if leaf == "conv_stem":
            layers.append(("stem", 224, 3, hh, c))
        elif leaf == "conv_dw":
            layers.append(("dw", act[0], act[1], hh, c))
        elif leaf.startswith("conv"):
            layers.append(("pw", act[0], act[1], hh, c))
        else:
            act = (hh, c)
    assert sum(k == "stem" for k, *_ in layers) == 2 and len(heads) == 2
    return layers, heads


def uniq(xs):
    return list(dict.fromkeys(xs))


# ---- BatchNorm forward ------------------------------------------------------------------------------------------------

def bn_forward(L, ws, z, C_, momentum=0.1, eps=1e-3, gamma=None, beta=None, rm=None, rv=None, nbt=0, res=None, relu=0, rnd=0):
    """-> (mean, invstd, y, running_mean, running_var, num_batches_tracked) after one smk_debug_train_bn_forward."""
    M = z.numel() // C_
    gamma = torch.ones(C_, device=DEV) if gamma is None else gamma
    beta = torch.zeros(C_, device=DEV) if beta is None else beta
    rm = torch.zeros(C_, device=DEV) if rm is None else rm.clone()
    rv = torch.ones(C_, device=DEV) if rv is None else rv.clone()
    n = torch.tensor([nbt], dtype=torch.int64, device=DEV)
    mean, invstd, y = torch.empty(C_, device=DEV), torch.empty(C_, device=DEV), torch.empty_like(z)
    m = -1.0 if momentum is None else momentum
    rc = L.smk_debug_train_bn_forward(P(z), M, C_, eps, m, P(gamma), P(beta), P(rm), P(rv), P(n), P(res), relu, rnd,
                                      P(mean), P(invstd), P(y), P(ws), ws.numel(), stream())
    assert rc == 0, L.smk_last_error()
    return mean, invstd, y, rm, rv, int(n.item())


def ref_stats(z, C_, eps):
    """fp64 batch mean, biased variance and 1 / sqrt(var + eps) (eps as the fp32 the kernel receives)."""
    z64 = z.view(-1, C_).double()
    M = z64.shape[0]
    mean = z64.sum(0) / M
    var = (z64 - mean).pow(2).sum(0) / M
    return mean, var, 1.0 / torch.sqrt(var + f32(eps))


def check_running(rm0, rv0, rm, rv, mean64, var64, M, momentum, nbt0, mean=None):
    """The update (1 - f) * r + f * batch, f = momentum or 1 / (num_batches_tracked + 1) (torch's momentum=None), the
    variance unbiased.  The fp32 evaluation rounds 1 - f, the two products, the fp32 batch value and the sum: at most
    3 u of s = |(1 - f) r| + |f batch|, inside the 2 ulp (4 u) of s allowed here.  Momentum 0 keeps the running
    statistics bitwise; momentum 1 replaces the running mean by the kernel's batch mean bitwise."""
    f = f32(momentum if momentum is not None else 1.0 / (nbt0 + 1))
    unb = var64 * M / (M - 1) if M > 1 else var64
    worst = 0.0
    for r0, r, batch in ((rm0, rm, mean64), (rv0, rv, unb)):
        a, b = (1 - f) * r0.double(), f * batch
        s = a.abs() + b.abs()
        err = ((r.double() - (a + b)).abs() / (4 * U * s).clamp_min(1e-300)).max().item()
        worst = max(worst, err)
        assert err <= 1.0, (momentum, nbt0, err)
    if momentum == 0:
        assert same(rm, rm0) and same(rv, rv0)
    if momentum == 1:
        assert same(rm, mean)
    return worst


def bn_shapes(topo, B):
    return uniq((B * ho * ho, co) for _, _, _, ho, co in topo[0])


BN_EDGES = [(999, 20), (1000, 24), (4096 + 8, 480), (1568, 576), (2000, 672), (1568, 960), (131071, 16), (131072, 16),
            (131073, 20), (153100, 16), (153100, 960)]


@pytest.mark.parametrize("B", [1, 32, None])
def test_bn_statistics_exact_on_integers(L, ws, topo, B):
    """Every BN shape of both backbones (None: the forced edges: M not a multiple of 8 / 16 / 256, C not a multiple of
    32 / 64 and C > 256 in the one-CTA finalize, M just below / at / above 131072 where the chunk count caps at 512, and
    M = 153100 where the 512th chunk is empty): mean bitwise, invstd within 1 ulp, running statistics of the update."""
    shapes = BN_EDGES if B is None else bn_shapes(topo, B)
    for i, (M, C_) in enumerate(shapes):
        if B is None and M > 131072:
            nch, chunk = MAX_CHUNKS, cdiv(M, MAX_CHUNKS)
            assert M == 131073 or (nch - 1) * chunk >= M          # 153100: the last chunk holds no pixel
        z = ints((M, C_), 100 + i)
        rm0, rv0 = randn(C_, 200 + i) * 0.1, randn(C_, 300 + i).abs() + 0.5
        mean, invstd, y, rm, rv, n = bn_forward(L, ws, z, C_, rm=rm0, rv=rv0, nbt=5)
        mean64, var64, inv64 = ref_stats(z, C_, 1e-3)
        assert same(mean, mean64.float()), (M, C_)
        assert (invstd.double() - inv64.float().double()).abs().le(ulp(inv64.float())).all(), (M, C_)
        check_running(rm0, rv0, rm, rv, mean64, var64, M, 0.1, 5)
        assert n == 6
        again = bn_forward(L, ws, z, C_, rm=rm0, rv=rv0, nbt=5)
        assert all(same(a, b) for a, b in zip((mean, invstd, y, rm, rv), again[:5])), (M, C_)


@pytest.mark.parametrize("momentum", [0.1, 0.0, 1.0, None])
def test_bn_running_statistics_update(L, ws, momentum):
    """momentum 0.1, 0 (running statistics unchanged bitwise), 1 (replaced by the batch's bitwise) and None (cumulative
    average, 1 / (num_batches_tracked + 1)), with the counter at 0, 5 and 2^40 (it is int64 on both sides), at
    C = 960 > 256 and M = 153100 (an empty last chunk)."""
    M, C_ = 153100, 960
    z = randn((M, C_), 7) * 2 + 0.5
    rm0, rv0 = randn(C_, 8) * 0.1, randn(C_, 9).abs() + 0.5
    mean64, var64, _ = ref_stats(z, C_, 1e-3)
    worst = 0.0
    for nbt in (0, 5, 1 << 40):
        mean, _, _, rm, rv, n = bn_forward(L, ws, z, C_, momentum=momentum, rm=rm0, rv=rv0, nbt=nbt)
        assert n == nbt + 1
        worst = max(worst, check_running(rm0, rv0, rm, rv, mean64, var64, M, momentum, nbt, mean))
    print("momentum %s: running statistics, worst error %.2f of the 2-ulp bound" % (momentum, worst))


def test_bn_statistics_hold_up_far_from_zero(L, ws):
    """|mean| / std ~ 1e3: the kernels form the variance as sum(z^2) / M - mean^2 in fp64, which cancels about 6 of its
    16 digits here and so still lands within an fp32 ulp or two; mean within 1 ulp (the fp64 sums are no longer exact)."""
    worst = [0.0, 0.0]
    for M, C_ in ((401408, 16), (25088, 240), (153100, 960)):
        z = randn((M, C_), 11) + 1000.0 * (1 + torch.arange(C_, device=DEV) % 3)
        mean, invstd, *_ = bn_forward(L, ws, z, C_)
        mean64, _, inv64 = ref_stats(z, C_, 1e-3)
        em = ((mean.double() - mean64).abs() / ulp(mean64.float())).max().item()
        ei = ((invstd.double() - inv64).abs() / ulp(inv64.float())).max().item()
        worst = [max(worst[0], em), max(worst[1], ei)]
        assert em <= 1.0 and ei <= 2.0, (M, C_, em, ei)
    print("|mean|/std ~ 1e3: mean %.2f ulp, invstd %.2f ulp" % tuple(worst))


@pytest.mark.parametrize("relu,use_res,rnd", [(1, 0, 0), (0, 1, 0), (1, 0, 1), (0, 1, 1)])
def test_bn_apply_on_random_data(L, ws, relu, use_res, rnd):
    """y = gamma * (z - mean) * invstd + beta (+ res) (ReLU) against fp64 with the kernel's own mean and invstd.  The fp32
    evaluation rounds z - mean, the two products, + beta and + res: at most 5 u of S = |xhat gamma| + |beta| + |res|,
    allowed 6 u.  With TF32 rounding (precision 1): the low 13 mantissa bits are zero and the rounding (to nearest)
    adds at most 2^-11 of the fp32 value, i.e. 2^-11 |ref| + 2^-11 * 6 u S, allowed 2^-11 |ref| + u S."""
    worst = 0.0
    for i, (M, C_) in enumerate(((999, 20), (25088, 240), (1568, 960))):
        z = randn((M, C_), 20 + i) * 3 + 1
        gamma, beta = randn(C_, 30 + i).abs() + 0.5, randn(C_, 40 + i) * 0.1
        res = randn((M, C_), 50 + i) if use_res else None
        mean, invstd, y, *_ = bn_forward(L, ws, z, C_, gamma=gamma, beta=beta, res=res, relu=relu, rnd=rnd)
        xh = (z.double() - mean.double()) * invstd.double()
        ref = xh * gamma.double() + beta.double() + (res.double() if use_res else 0)
        S = (xh * gamma.double()).abs() + beta.double().abs() + (res.double().abs() if use_res else 0)
        if relu:
            ref = ref.clamp_min(0)
        tol = 6 * U * S
        if rnd:
            assert (y.view(torch.int32) & 0x1FFF).eq(0).all(), "outputs not TF32-rounded"
            tol = tol + U * S + 2.0 ** -11 * ref.abs()
        err = ((y.double() - ref).abs() / tol.clamp_min(1e-300)).max().item()
        worst = max(worst, err)
        assert err <= 1.0, (M, C_, err)
    print("bn apply relu %d res %d round %d: worst error %.2f of the bound" % (relu, use_res, rnd, worst))


# ---- BatchNorm backward -----------------------------------------------------------------------------------------------

def bn_backward(L, ws, g, y, z, mean, invstd, gamma, C_, rnd=0, gz=None):
    M = z.numel() // C_
    gz = torch.empty_like(g) if gz is None else gz
    gg, gb = torch.empty(C_, device=DEV), torch.empty(C_, device=DEV)
    rc = L.smk_debug_train_bn_backward(P(g), P(y), P(z), P(mean), P(invstd), P(gamma), M, C_, rnd, P(gz), P(gg), P(gb), P(ws), ws.numel(),
                                       stream())
    assert rc == 0, L.smk_last_error()
    return gz, gg, gb


@pytest.mark.parametrize("B", [1, 32, None])
def test_bn_backward_exact_sums_and_g_z(L, ws, topo, B):
    """g_beta = sum g' bitwise (g' = g [y > 0]; integer g); g_gamma within 1 ulp of the fp64 sum of g' * xhat, xhat the
    kernel's own fp32 (z - mean) * invstd; g_z against fp64 from the kernel's sums: rounding 1 / M, the two scaled sums,
    xhat times one, the two differences and the two products is at most 8 u of
    S = |gamma invstd| (|g'| + |g_beta / M| + |xhat g_gamma / M|).  In place (g_z aliasing g) equals out of place
    bitwise, and a second launch repeats bitwise."""
    shapes = BN_EDGES if B is None else bn_shapes(topo, B)
    worst = 0.0
    for i, (M, C_) in enumerate(shapes):
        z = randn((M, C_), 400 + i) * 2 + 0.3
        mean64, _, inv64 = ref_stats(z, C_, 1e-3)
        mean, invstd = mean64.float(), inv64.float()
        gamma = randn(C_, 500 + i).abs() + 0.5
        g = ints((M, C_), 600 + i)
        for y in (None, torch.relu(ints((M, C_), 700 + i))):
            gz, gg, gb = bn_backward(L, ws, g, y, z, mean, invstd, gamma, C_)
            gp = g.double() if y is None else g.double() * (y > 0)
            xh = ((z - mean) * invstd).double()                    # fp32, as the kernel forms it
            assert same(gb, gp.sum(0).float()), (M, C_)
            assert (gg.double() - (gp * xh).sum(0).float().double()).abs().le(ulp((gp * xh).sum(0).float())).all(), (M, C_)
            k = (gamma.double() * invstd.double())
            ref = k * (gp - gb.double() / M - xh * (gg.double() / M))
            S = k.abs() * (gp.abs() + (gb.double() / M).abs() + (xh * gg.double() / M).abs())
            err = ((gz.double() - ref).abs() / (8 * U * S).clamp_min(1e-300)).max().item()
            worst = max(worst, err)
            assert err <= 1.0, (M, C_, y is None, err)
            inplace = g.clone()
            bn_backward(L, ws, inplace, y, z, mean, invstd, gamma, C_, gz=inplace)
            assert same(inplace, gz), (M, C_)
            again = bn_backward(L, ws, g, y, z, mean, invstd, gamma, C_)
            assert all(same(a, b) for a, b in zip((gz, gg, gb), again))
    print("bn backward B %s: g_z worst error %.2f of the bound" % (B, worst))


# ---- weight gradients -------------------------------------------------------------------------------------------------

def wgrad_chunks(M, tiles, tile_floats, per_chunk_min):
    """encoder_train.cu's wgrad_chunks -> (chunks, the bound that chose them: 'pixels', 'tiles' or 'cap')."""
    cands = {"pixels": cdiv(M, per_chunk_min), "tiles": 1024 // tiles + 1, "cap": max(1, WGRAD_PART // (tiles * tile_floats))}
    which = min(cands, key=lambda k: (cands[k], ["pixels", "tiles", "cap"].index(k)))
    return max(1, cands[which]), which


def pw_wgrad(L, ws, g, a, Co, Ci):
    M = g.numel() // Co
    out = torch.empty(Co, Ci, device=DEV)
    rc = L.smk_debug_train_pw_wgrad(P(g), P(a), M, Co, Ci, P(out), P(ws), ws.numel(), stream())
    assert rc == 0, L.smk_last_error()
    return out


def pw_shapes(topo, B):
    return uniq((B * ho * ho, co, ci) for k, _, ci, ho, co in topo[0] if k == "pw")


PW_EDGES = [(1000, 72, 24), (999, 960, 160), (1568, 160, 960), (25088, 40, 120), (613700, 16, 16), (401408, 96, 16)]


@pytest.mark.parametrize("B", [1, 32, None])
def test_pw_wgrad_exact_on_integers(L, ws, topo, B):
    """Bitwise on integers at every 1x1 shape, and at the edges: Co / Ci tails of the 64 x 64 tile (72 x 24,
    960 x 160, 160 x 960), M not a multiple of 16, both chunk bounds of wgrad_chunks (pixels; the partial-buffer cap),
    and M = 613700, where the 1024th chunk is empty."""
    shapes = PW_EDGES if B is None else pw_shapes(topo, B)
    seen = set()
    for i, (M, Co, Ci) in enumerate(shapes):
        tiles = cdiv(Ci, 64) * cdiv(Co, 64)
        nch, which = wgrad_chunks(M, tiles, 64 * 64, 512)
        seen.add(which)
        if M == 613700:
            assert nch == 1024 and (nch - 1) * cdiv(M, nch) >= M
        g, a = ints((M, Co), 800 + i), ints((M, Ci), 900 + i)
        out = pw_wgrad(L, ws, g, a, Co, Ci)
        assert same(out, (g.double().t() @ a.double()).float()), (M, Co, Ci, nch)
        assert same(out, pw_wgrad(L, ws, g, a, Co, Ci))
    if B is None:
        assert seen == {"pixels", "cap"}, seen      # 'tiles' never binds here: the cap is floor(1024 / tiles)


def test_weight_gradients_on_random_data(L, ws):
    """Random fp32 against fp64.  Within a chunk the kernels accumulate n = chunk pixels in fp32, whose rounding errors
    grow like sqrt(n) u of the partial sums; the chunks are summed in fp64.  Bound: 8 sqrt(n) u of max |ref|."""
    worst = 0.0
    for i, (M, Co, Ci) in enumerate(((1000, 72, 24), (25088, 40, 120), (1568, 960, 160), (401408, 96, 16))):
        g, a = randn((M, Co), 1000 + i), randn((M, Ci), 1100 + i)
        out = pw_wgrad(L, ws, g, a, Co, Ci)
        ref = g.double().t() @ a.double()
        n = cdiv(M, wgrad_chunks(M, cdiv(Ci, 64) * cdiv(Co, 64), 4096, 512)[0])
        err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
        worst = max(worst, err)
        assert err <= 8 * n ** 0.5 * U, (M, Co, Ci, err)
    for i, (B, H, C_, S) in enumerate(((32, 112, 16, 1), (32, 28, 480, 1), (2, 15, 72, 2))):
        g, a = randn((B, cdiv(H, S), cdiv(H, S), C_), 1200 + i), randn((B, H, H, C_), 1300 + i)
        out = dw_wgrad(L, ws, g, a, B, H, C_, S)
        ref = dw_ref(a, g, None, S)[2]
        M = B * cdiv(H, S) ** 2
        n = cdiv(M, min(wgrad_chunks(M, cdiv(C_, 32), 32 * 9, 256)[0], 256))
        err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
        worst = max(worst, err)
        assert err <= 8 * n ** 0.5 * U, (B, H, C_, S, err)
    img, g = randn((32, 3, 224, 224), 1400), randn((32, 112, 112, 16), 1401)
    out = stem_wgrad(L, ws, g, img)
    ref = stem_ref(img, None, g)[1]
    err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    worst = max(worst, err)
    assert err <= 8 * 1024 ** 0.5 * U, err
    print("weight gradients on random data: worst max-abs error / max-abs %.2e" % worst)


# ---- depthwise ----------------------------------------------------------------------------------------------------------

def same_pad(H, S):
    Ho = cdiv(H, S)
    total = max((Ho - 1) * S + 3 - H, 0)
    return total // 2, total - total // 2


def dw_ref(a, g, w, S, res=None):
    """fp64 TF-SAME depthwise conv of a [B,H,H,C] NHWC (w [C,1,3,3]) -> (z, g_a, g_w) (NHWC; None where not asked)."""
    x = a.permute(0, 3, 1, 2).double().requires_grad_()
    C_ = x.shape[1]
    wd = (w.double() if w is not None else torch.zeros(C_, 1, 3, 3, dtype=torch.float64, device=DEV)).requires_grad_()
    b, e = same_pad(x.shape[2], S)
    z = F.conv2d(F.pad(x, (b, e, b, e)), wd, stride=S, groups=C_)
    if g is None:
        return z.permute(0, 2, 3, 1), None, None
    ga, gw = torch.autograd.grad(z, (x, wd), g.permute(0, 3, 1, 2).double())
    ga = ga.permute(0, 2, 3, 1) + (res.double() if res is not None else 0)
    return z.detach().permute(0, 2, 3, 1), ga, gw


def dw_forward(L, a, w, B, H, C_, S):
    z = torch.empty(B, cdiv(H, S), cdiv(H, S), C_, device=DEV)
    assert L.smk_debug_train_dw_forward(P(a), P(w), B, H, C_, S, P(z), stream()) == 0, L.smk_last_error()
    return z


def dw_wgrad(L, ws, g, a, B, H, C_, S):
    out = torch.empty(C_, 1, 3, 3, device=DEV)
    assert L.smk_debug_train_dw_wgrad(P(g), P(a), B, H, C_, S, P(out), P(ws), ws.numel(), stream()) == 0, L.smk_last_error()
    return out


def dw_dgrad(L, g, w, res, B, H, C_, S):
    out = torch.empty(B, H, H, C_, device=DEV)
    assert L.smk_debug_train_dw_dgrad(P(g), P(w), P(res), B, H, C_, S, P(out), stream()) == 0, L.smk_last_error()
    return out


DW_EDGES = [(2, 15, 72, 2), (2, 14, 72, 2), (3, 7, 200, 2), (1, 9, 20, 1), (32, 28, 480, 1), (32, 112, 16, 1)]


@pytest.mark.parametrize("B", [1, 32, None])
def test_depthwise_exact_on_integers(L, ws, topo, B):
    """Forward, dgrad (with and without the skip residual) and weight gradient bitwise on integers at every depthwise
    shape, and at the edges: stride 2 at odd and even H (TF-SAME pads the odd row after), C not a multiple of 32, and
    the three bounds of the weight gradient's chunk count (pixels, tiles, the 256-chunk cap)."""
    shapes = DW_EDGES if B is None else uniq((B, hi, c, 1 if ho == hi else 2) for k, hi, c, ho, _ in topo[0] if k == "dw")
    seen = set()
    for i, (B_, H, C_, S) in enumerate(shapes):
        Ho = cdiv(H, S)
        M = B_ * Ho * Ho
        nch, which = wgrad_chunks(M, cdiv(C_, 32), 32 * 9, 256)
        seen.add("cap256" if nch > 256 else which)
        a, w = ints((B_, H, H, C_), 1500 + i), ints((C_, 1, 3, 3), 1600 + i)
        g, res = ints((B_, Ho, Ho, C_), 1700 + i), ints((B_, H, H, C_), 1800 + i)
        z_ref, ga_ref, gw_ref = dw_ref(a, g, w, S, res)
        assert same(dw_forward(L, a, w, B_, H, C_, S), z_ref.float()), (B_, H, C_, S)
        assert same(dw_dgrad(L, g, w, res, B_, H, C_, S), ga_ref.float()), (B_, H, C_, S)
        assert same(dw_dgrad(L, g, w, None, B_, H, C_, S), (ga_ref - res.double()).float()), (B_, H, C_, S)
        gw = dw_wgrad(L, ws, g, a, B_, H, C_, S)
        assert same(gw, gw_ref.float()), (B_, H, C_, S, nch)
        assert same(gw, dw_wgrad(L, ws, g, a, B_, H, C_, S))
    if B is None:
        assert seen == {"pixels", "tiles", "cap256"}, seen


# ---- stem ---------------------------------------------------------------------------------------------------------------

def stem_ref(img, w, g=None):
    x = img.double().requires_grad_()
    wd = (w.double() if w is not None else torch.zeros(16, 3, 3, 3, dtype=torch.float64, device=DEV)).requires_grad_()
    b, e = same_pad(x.shape[2], 2)
    b2, e2 = same_pad(x.shape[3], 2)
    z = F.conv2d(F.pad(x, (b2, e2, b, e)), wd, stride=2)
    if g is None:
        return z.detach().permute(0, 2, 3, 1), None
    return None, torch.autograd.grad(z, wd, g.permute(0, 3, 1, 2).double())[0]


def stem_wgrad(L, ws, g, img):
    B, _, H, W = img.shape
    out = torch.empty(16, 3, 3, 3, device=DEV)
    assert L.smk_debug_train_stem_wgrad(P(g), P(img), B, H, W, P(out), P(ws), ws.numel(), stream()) == 0, L.smk_last_error()
    return out


@pytest.mark.parametrize("B,H,W", [(1, 224, 224), (32, 224, 224), (48, 224, 224), (3, 15, 17), (2, 30, 18)])
def test_stem_exact_on_integers(L, ws, B, H, W):
    """Stem conv and its weight gradient bitwise on integers: the train shape at B = 1, 32 and 48 (M = 602112 > 524288:
    the 512-chunk cap), and small odd and even images."""
    img, w = ints((B, 3, H, W), 1900 + B), ints((16, 3, 3, 3), 2000 + B)
    Ho, Wo = cdiv(H, 2), cdiv(W, 2)
    z = torch.empty(B, Ho, Wo, 16, device=DEV)
    assert L.smk_debug_train_stem_forward(P(img), P(w), B, H, W, P(z), stream()) == 0, L.smk_last_error()
    assert same(z, stem_ref(img, w)[0].float())
    g = ints((B, Ho, Wo, 16), 2100 + B)
    gw = stem_wgrad(L, ws, g, img)
    assert same(gw, stem_ref(img, None, g)[1].float())
    assert same(gw, stem_wgrad(L, ws, g, img))
    if B == 48:
        assert cdiv(B * Ho * Wo, 1024) > 512


# ---- head ---------------------------------------------------------------------------------------------------------------

def test_head_backward_masks_and_gradients(L, topo):
    """The clamp / ReLU masks against torch's own backward on the same fp32 values, with values placed exactly on 0, 1,
    -0.2f and 0.2f and one ulp either side; then g_feat = W^T gp / HW, g_W and g_b bitwise on integers (the sums are
    exact and the division is correctly rounded on both sides)."""
    import itertools
    B, HW = 4, 49
    for (feat, n_out), use_codes in itertools.product(topo[1] + [(960, 55)], (True, False)):
        codes = ints((n_out,), n_out, 0, 3).to(torch.uint8) if use_codes else None
        edges = torch.tensor([0.0, 1.0, -0.2, 0.2], dtype=torch.float32, device=DEV)
        pts = torch.cat([edges, torch.nextafter(edges, edges + 1), torch.nextafter(edges, edges - 1)])
        raw = randn((B, n_out), n_out) * 0.6 + 0.3
        flat = raw.view(-1)
        sel = torch.arange(0, flat.numel(), 2, device=DEV)      # every other value on an edge, each edge under every code
        flat[sel] = pts[(sel // 2) % pts.numel()]
        g = ints((B, n_out), 2200 + n_out, 1, 2)                # non-zero: a masked value shows as a zero in gp
        w, pooled = ints((n_out, feat), 2300 + n_out), ints((B, feat), 2400 + n_out)
        gp, gy = torch.empty(B, n_out, device=DEV), torch.empty(B, HW, feat, device=DEV)
        gw, gb = torch.empty(n_out, feat, device=DEV), torch.empty(n_out, device=DEV)
        rc = L.smk_debug_train_head_backward(P(g), P(raw), P(codes), P(w), P(pooled), B, n_out, HW, feat, P(gp), P(gy), P(gw), P(gb),
                                             stream())
        assert rc == 0, L.smk_last_error()
        x = raw.clone().requires_grad_()
        outs = [x, torch.clamp(x, 0, 1), torch.relu(x), torch.clamp(x, -0.2, 0.2)]
        code = codes.long() if use_codes else torch.zeros(n_out, dtype=torch.long, device=DEV)
        y = torch.stack(outs).gather(0, code.view(1, 1, -1).expand(1, B, n_out))[0]
        want = torch.autograd.grad(y, x, g)[0]
        assert same(gp, want), (n_out, use_codes)
        want_feat = (want.double() @ w.double() / HW).float()   # an integer / 49 is never near an fp32 tie: rounds once
        assert same(gy, want_feat[:, None, :].expand(B, HW, feat).contiguous())
        assert same(gw, (want.double().t() @ pooled.double()).float()) and same(gb, want.double().sum(0).float())


# ---- per-layer audit of the real train forward --------------------------------------------------------------------------

def _encoder(precision):
    import smirk_b200
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    enc = enc.to(DEV).train().allow_train_mode_(True)
    for m in enc.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = 0.1
        if hasattr(m, "precision"):
            m.precision = precision
    return enc


@pytest.mark.parametrize("B,precision", [(32, 0), (32, 3), (1, 0)])
def test_per_layer_audit_of_the_train_forward(native_lib, B, precision):
    """One train forward (with the running-statistics update); every layer checked from the device's own saved input:
    the pre-BN output of each conv against an fp64 conv (of max |ref|: 1e-5 for fp32, 4e-6 sqrt(K / 64) for the 3xTF32
    1x1 convs, as in test_gpu_kernels.py), the batch statistics against fp64 statistics of the saved z (1e-6), each ReLU / block output
    against fp64 BatchNorm of the saved z with the device's statistics plus the saved skip input (1e-6 of max |ref|),
    and each module's running statistics against the fp64 update (1e-6 of the update's scale)."""
    from smirk_b200 import _lib
    enc = _encoder(precision)
    img = synth_inputs.images(B, 2500 + B).to(DEV)
    parts = (enc.pose_encoder, enc.shape_encoder, enc.expression_encoder)
    bns, convs = [], []
    for p in parts:
        bns += [m for m in p.encoder.modules() if isinstance(m, nn.BatchNorm2d)]
        convs += [m for m in p.encoder.modules() if isinstance(m, nn.Conv2d)]
    before = [(m.running_mean.clone(), m.running_var.clone(), int(m.num_batches_tracked)) for m in bns]
    with torch.no_grad():
        h, _, saved = enc._forward_train(img, enc._train_params(), True)
    views = _lib.saved_views("encoder", h, saved, B)
    # the statistics follow the saved tensors, each of which is padded to a multiple of 64 floats per image
    stats = saved[max(v.storage_offset() + B * cdiv(v.numel() // B, 64) * 64 for v in views.values()):]
    errs = {"z": 0.0, "stats": 0.0, "y": 0.0, "running": 0.0}
    k, off, act, block, block_in, z = 0, 0, None, None, None, None
    x_img = img.double()
    for name, v in views.items():
        if v.dim() == 2:
            continue
        leaf = name.rsplit(".", 1)[1]
        if leaf.startswith("conv"):
            conv, bn = convs[k], bns[k]
            C_ = v.shape[1]
            assert conv.out_channels == C_ == bn.num_features, name
            prefix = name.rsplit(".", 1)[0]
            if prefix != block:
                block, block_in = prefix, act
            w = conv.weight.double()
            if leaf == "conv_stem":
                b, e = same_pad(224, 2)
                ref = F.conv2d(F.pad(x_img, (b, e, b, e)), w, stride=2)
            elif leaf == "conv_dw":
                S = 1 if act.shape[2] == v.shape[2] else 2
                b, e = same_pad(act.shape[2], S)
                ref = F.conv2d(F.pad(act.double(), (b, e, b, e)), w, stride=S, groups=C_)
            else:
                ref = F.conv2d(act.double(), w)
            errs["z"] = max(errs["z"], e_z := ((v.double() - ref).abs().max() / ref.abs().max()).item())
            x3 = precision == 3 and leaf not in ("conv_stem", "conv_dw")
            assert e_z <= (4e-6 * max(1.0, (conv.in_channels / 64) ** 0.5) if x3 else 1e-5), (name, e_z)
            z = v.double()
            M = z.numel() // C_
            mean_d, inv_d = stats[off:off + C_].double(), stats[off + C_:off + 2 * C_].double()
            off += 2 * C_
            mean64 = z.sum((0, 2, 3)) / M
            var64 = (z - mean64.view(1, -1, 1, 1)).pow(2).sum((0, 2, 3)) / M
            inv64 = 1.0 / torch.sqrt(var64 + f32(bn.eps))
            e_s = max(((mean_d - mean64).abs() / (mean64.abs() + var64.sqrt())).max().item(),
                      ((inv_d - inv64).abs() / inv64).max().item())
            errs["stats"] = max(errs["stats"], e_s)
            assert e_s <= 1e-6, (name, e_s)
            rm0, rv0, n0 = before[k]
            f = bn.momentum
            for r0, r, batch in ((rm0, bn.running_mean, mean64), (rv0, bn.running_var, var64 * M / max(M - 1, 1))):
                want = (1 - f) * r0.double() + f * batch
                e_r = ((r.double() - want).abs() / ((1 - f) * r0.double().abs() + f * batch.abs()).clamp_min(1e-30)).max().item()
                errs["running"] = max(errs["running"], e_r)
                assert e_r <= 1e-6, (name, e_r)
            assert int(bn.num_batches_tracked) == n0 + 1
            k += 1
            cur = (bn.weight.double(), bn.bias.double(), mean_d, inv_d)
        else:
            gam, bet, mean_d, inv_d = cur
            sh = lambda t: t.view(1, -1, 1, 1)
            ref = (z - sh(mean_d)) * sh(inv_d) * sh(gam) + sh(bet)
            relu = leaf.startswith("bn")
            if not relu and block_in is not None and block_in.shape == v.shape:
                ref = ref + block_in.double()
            if relu:
                ref = ref.clamp_min(0)
            errs["y"] = max(errs["y"], e_y := ((v.double() - ref).abs().max() / ref.abs().max()).item())
            assert e_y <= 1e-6, (name, e_y)
            act = v
    assert k == len(bns) == len(convs) and off <= stats.numel()
    print("per-layer audit B %d precision %d over %d layers: z %.2e, stats %.2e, outputs %.2e, running stats %.2e"
          % (B, precision, k, errs["z"], errs["stats"], errs["y"], errs["running"]))
