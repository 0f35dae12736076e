"""GPU suite (-m gpu): steady-state hand-offs of the fused expand 1x1 + depthwise 3x3 kernel (xdw_tc.cu).

test_gpu_xdw_window.py runs B = 2, where most persistent CTAs see one or two work items.  Here B = 32 makes every CTA walk
many items, so the E ring, the weight ring and the window buffers wrap across item boundaries many times; B = 1 splits one
image's channel chunks over many CTAs.  On small integers every product and sum is exact in TF32 and fp32, so the output must
equal the CPU result bit for bit, and a second launch on the same input must reproduce the first."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_xdw_window import LAYERS, run, tf_same_dw

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 32])
@pytest.mark.parametrize("x3", [0, 1], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("H,Cin,mid,stride", LAYERS)
def test_xdw_steady_state_exact(native_lib, H, Cin, mid, stride, x3, B):
    g = torch.Generator().manual_seed(3000 * H + Cin + mid + stride + B)
    x = torch.randint(-2, 3, (B, Cin, H, H), generator=g).float()
    w1 = torch.randint(-1, 2, (mid, Cin, 1, 1), generator=g).float()
    wd = torch.randint(-1, 2, (mid, 1, 3, 3), generator=g).float()
    one, zero = torch.ones(mid), torch.zeros(mid)
    ref = F.relu(tf_same_dw(F.relu(F.conv2d(x.double(), w1.double())), wd.double(), stride)).float()
    got = run(native_lib, x3, x, w1, one, zero, wd, one, zero, stride)
    assert torch.equal(got, ref), "%d of %d outputs differ" % (int((got != ref).sum()), ref.numel())
    again = run(native_lib, x3, x, w1, one, zero, wd, one, zero, stride)
    assert torch.equal(again, got), "second launch differs in %d outputs" % int((again != got).sum())
