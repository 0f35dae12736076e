"""GPU suite (-m gpu): the fused expand 1x1 + depthwise 3x3 kernel (xdw_tc.cu) on sizes whose output tiles are ragged.

A depthwise thread covers a channel quad x a short run of adjacent output columns x a run of rows; the runs are cut from the
tile's column and row counts and the number of depthwise threads of each schedule.  These sizes give edge tiles of odd and
small widths: stride 1 at H = 9 (one 9-column tile), 15 (14 + 1) and 20 (14 + 6); stride 2 at H = 18 (7 + 2 outputs) and 30
(7 + 7 + 1).  The two channel widths give a partial last chunk (72 = 2 x 32 + 8) and a full one with Cin past one k-block.
On small integers every product and sum is exact, so both entry points (plain TF32 and 3xTF32) must equal the CPU result bit
for bit, and a second launch must reproduce the first."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_xdw_window import run, tf_same_dw

pytestmark = pytest.mark.gpu

RAGGED = [(9, 1), (15, 1), (20, 1), (18, 2), (30, 2)]


@pytest.mark.parametrize("B", [1, 32])
@pytest.mark.parametrize("x3", [0, 1], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("Cin,mid", [(16, 72), (40, 128)])
@pytest.mark.parametrize("H,stride", RAGGED)
def test_xdw_ragged_tiles_exact(native_lib, H, stride, Cin, mid, x3, B):
    g = torch.Generator().manual_seed(4000 * H + Cin + mid + stride + B)
    x = torch.randint(-2, 3, (B, Cin, H, H), generator=g).float()
    w1 = torch.randint(-1, 2, (mid, Cin, 1, 1), generator=g).float()
    wd = torch.randint(-1, 2, (mid, 1, 3, 3), generator=g).float()
    one, zero = torch.ones(mid), torch.zeros(mid)
    ref = F.relu(tf_same_dw(F.relu(F.conv2d(x.double(), w1.double())), wd.double(), stride)).float()
    got = run(native_lib, x3, x, w1, one, zero, wd, one, zero, stride)
    assert torch.equal(got, ref), "%d of %d outputs differ" % (int((got != ref).sum()), ref.numel())
    again = run(native_lib, x3, x, w1, one, zero, wd, one, zero, stride)
    assert torch.equal(again, got), "second launch differs in %d outputs" % int((again != got).sum())
