"""The 128-wide N tile of the forward / data-gradient kernel on a stride-2 convolution: its data gradient scatters
the output rows with stride 2, which the small-batch cases of test_gpu_conv_tc.py reach only through the K-split,
64-wide path."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from eventgrad_b200.ops import conv_tc, ext  # noqa: E402


def test_stride2_data_gradient_on_the_wide_tile_matches_fp64():
    N, H, Ci, Co = 160, 16, 128, 256
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # every parity class of the data gradient (1, 2, 2, 4 taps over dY) runs 128 wide (80 tiles on an H100)
    for taps in (1, 2, 4):
        assert ext().conv_fprop_ntile(N, H // 2, H // 2, Co, Ci, taps, sms) == 128
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(N, Ci, H, H, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) * (2.0 / (9 * Ci)) ** 0.5).contiguous(
        memory_format=torch.channels_last)
    assert conv_tc.kind_of(x, w, (2, 2), (1, 1), (1, 1), 1) == "s2"
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, stride=2, padding=1)
    dy = torch.randn(yd.shape, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    yd.backward(dy.double())
    x1, w1 = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y1 = conv_tc.conv2d(x1, w1, None, (2, 2), (1, 1), (1, 1), 1)
    y1.backward(dy)
    for name, ours, truth in (("y", y1, yd), ("dx", x1.grad, xd.grad), ("dw", w1.grad, wd.grad)):
        truth = truth.detach()
        rms = float(((ours.double() - truth) ** 2).mean().sqrt() / (truth ** 2).mean().sqrt())
        rel = float((ours.double() - truth).abs().max() / truth.abs().max())
        assert ours.shape == truth.shape, name
        assert rms < 5e-7 and rel < 4e-6, (name, rms, rel)
