"""GPU suite for the generator train path's 3x3 weight gradient, one call at a time through smk_debug_train_conv3_wgrad
(the host helper the train backward runs): every 3x3 layer shape of the (6, 3, 32, 5) generator at B = 1 and 32, zero and
reflection padding, an input read with a pixel stride wider than its channels (a concat slice), and the shapes where the
split-K chunk count changes, against torch in float64 (max-abs error over max-abs <= 1e-5); on small integers, where
every partial sum is exact in fp32, bit for bit."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (cin, cout, S, reflect, lda) of every 3x3 conv of SmirkGenerator(6, 3, 32, 5); lda: the input's pixel stride (fp32 path)
F = 32
LAYERS = ([(6, F, 224, 0, 8), (F, F, 224, 0, F)]
          + [(F << (l - 1), F << l, 224 >> l, 0, F << (l - 1)) for l in (1, 2, 3, 4)]
          + [(F << l, F << l, 224 >> l, 0, F << l) for l in (1, 2, 3, 4)]
          + [(16 * F, 16 * F, 14, 1, 16 * F)]
          + [(2 * (F << l), F << l, 224 >> l, 0, 2 * (F << l)) for l in (3, 2, 1, 0)])


def wgrad(g, a, cin, reflect):
    """Device weight gradient of g [B,H,W,cout] over a [B,H,W,lda] -> [cout][cin][3][3]."""
    from smirk_b200 import _lib
    B, H, W, cout = g.shape
    out = torch.empty(cout, cin, 3, 3, device=DEV)
    ws = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)
    _lib.call("smk_debug_train_conv3_wgrad", g.device, g, a, a.shape[3], B, H, W, cin, cout, reflect, out, ws, ws.numel())
    return out


def reference(g, a, cin, reflect):
    x = a[..., :cin].permute(0, 3, 1, 2).double()
    gy = g.permute(0, 3, 1, 2).double()
    if reflect:
        xp = torch.nn.functional.pad(x, (1, 1, 1, 1), mode="reflect")
        return torch.nn.grad.conv2d_weight(xp, (gy.shape[1], cin, 3, 3), gy, padding=0)
    return torch.nn.grad.conv2d_weight(x, (gy.shape[1], cin, 3, 3), gy, padding=1)


def _check(B, H, W, cin, cout, reflect, lda, seed, integer=False):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    if integer:
        g = torch.randint(-2, 3, (B, H, W, cout), generator=gen, device=DEV).float()
        a = torch.randint(-2, 3, (B, H, W, lda), generator=gen, device=DEV).float()
    else:
        g = torch.randn(B, H, W, cout, generator=gen, device=DEV)
        a = torch.randn(B, H, W, lda, generator=gen, device=DEV)
    got = wgrad(g, a, cin, reflect).double()
    ref = reference(g, a, cin, reflect)
    if integer:
        assert torch.equal(got, ref)
        return 0.0
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err <= 1e-5, err
    return err


@pytest.mark.parametrize("B", [1, 32])
@pytest.mark.parametrize("layer", LAYERS, ids=lambda l: "%dto%d_%d_r%d_ld%d" % l)
def test_every_layer_shape(native_lib, layer, B):
    cin, cout, S, reflect, lda = layer
    err = _check(B, S, S, cin, cout, reflect, lda, 7 + cin + S)
    print("%s B %d: %.2e" % (layer, B, err))


@pytest.mark.parametrize("reflect", [0, 1])
def test_both_paddings_and_a_strided_concat_slice(native_lib, reflect):
    _check(2, 28, 28, 64, 32, reflect, 128, 11)          # the first half of a 128-channel concat


@pytest.mark.parametrize("shape", [(1, 16, 32), (1, 19, 27), (2, 16, 16), (1, 4, 4), (3, 100, 60)])
@pytest.mark.parametrize("ch", [(8, 16), (72, 40), (512, 512)])
def test_chunk_count_edges(native_lib, shape, ch):
    """M = 512 and 513 pixels (one chunk / two), tiny and odd shapes, and layer widths with 1 to 576 output tiles."""
    B, H, W = shape
    cin, cout = ch
    if cin * cout > 64 * 64 and H * W * B > 2000:
        pytest.skip("large width at a large size is covered by the layer shapes")
    _check(B, H, W, cin, cout, 0, cin, 21)
    _check(B, H, W, cin, cout, 1, cin, 22)


@pytest.mark.parametrize("layer", [LAYERS[0], LAYERS[1], LAYERS[10], LAYERS[11]], ids=lambda l: "%dto%d_%d_r%d" % l[:4])
def test_small_integers_bitwise(native_lib, layer):
    cin, cout, S, reflect, lda = layer
    _check(2, S, S, cin, cout, reflect, lda, 31, integer=True)


def test_bad_arguments(native_lib):
    from smirk_b200 import _lib
    L = _lib.lib()
    assert L.smk_debug_train_conv3_wgrad(None, None, 8, 1, 4, 4, 8, 8, 0, None, None, 0, None) < 0
    assert b"null" in L.smk_last_error()
