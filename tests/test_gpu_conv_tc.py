"""wgmma fp32-accuracy 3x3 convolution (csrc/conv_tc.cu) against an fp64 convolution.

The claim under test: the tensor-core path (three bf16 planes per fp32 tensor, six MMAs per product, fp32
accumulation) is as accurate as cuDNN's native fp32 kernels.  Every case computes the TRUTH in fp64, measures
cuDNN-fp32's error against it, and requires ours to be within a small factor of that (and tiny in absolute terms).
Reference op: torch::nn::Conv2d(3x3, stride 1, pad 1, no bias) of /root/reference/dcifar10/common/resnet.hpp:3-9.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from eventgrad_b200.ops import conv_tc  # noqa: E402

CASES = [  # N, H, W, Cin, Cout
    (4, 32, 32, 64, 64),
    (4, 16, 16, 128, 128),
    (4, 16, 16, 64, 128),
    (6, 8, 8, 256, 256),
    (16, 4, 4, 512, 512),
    (5, 4, 4, 128, 64),      # 4x4 images, batch not a multiple of the 8-image tile: zero-filled tail
    (3, 8, 8, 64, 64),       # odd number of 2-image tiles
    (40, 32, 32, 64, 64),    # 320 tiles: persistent CTAs walk several tiles, no K split (the small cases above all split K)
    (40, 16, 16, 128, 128),  # un-split 16-wide, N tile 128
    (40, 16, 16, 128, 64),   # ... N tile 64, two channel blocks
    (37, 16, 16, 64, 128),   # ... odd image count, Cin != Cout (dgrad runs the other instantiation)
]


def _rel(a, truth):
    return float((a.double() - truth).abs().max() / truth.abs().max())


def _rms(a, truth):
    return float(((a.double() - truth) ** 2).mean().sqrt() / (truth ** 2).mean().sqrt())


def _bias(a, truth):
    """signed shrink towards zero, relative: > 0 means |a| < |truth| on average (tensor-core truncation shows here)"""
    return float(((truth - a.double()) * truth.sign()).mean() / truth.abs().mean())


def _mk(N, H, W, Ca, Cb, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, Ca, H, W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Cb, Ca, 3, 3, device="cuda", generator=g) * (2.0 / (9 * Ca)) ** 0.5).contiguous(
        memory_format=torch.channels_last)
    dy = torch.randn(N, Cb, H, W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    return x, w, dy


def test_split3_is_exact_to_2pow_minus_24():
    x = torch.randn(1 << 16, device="cuda") * torch.logspace(-6, 6, 1 << 16, device="cuda")
    p = conv_tc.split3(x).float()
    back = (p[2].double() + p[1].double() + p[0].double())
    err = ((back - x.double()).abs() / x.double().abs().clamp_min(1e-30)).max()
    assert float(err) <= 2.0 ** -23, float(err)
    assert torch.equal(p[0], x.to(torch.bfloat16).float())


@pytest.mark.parametrize("N,H,W,Ca,Cb", CASES)
def test_forward_matches_fp64(N, H, W, Ca, Cb):
    torch.backends.cudnn.allow_tf32 = False
    x, w, _ = _mk(N, H, W, Ca, Cb)
    assert conv_tc.eligible(x, w, (1, 1), (1, 1), (1, 1), 1)
    truth = F.conv2d(x.double(), w.double(), padding=1)
    ours = conv_tc.conv3x3_tc(x, w)
    ref32 = F.conv2d(x, w, padding=1)
    assert ours.shape == ref32.shape and ours.is_contiguous(memory_format=torch.channels_last)
    e_ours, e_ref = _rms(ours, truth), _rms(ref32, truth)
    print(f"fwd {N}x{H}x{W} {Ca}->{Cb}: rms err ours {e_ours:.3e} cudnn-fp32 {e_ref:.3e} | max ours {_rel(ours, truth):.3e} "
          f"cudnn {_rel(ref32, truth):.3e} | shrink ours {_bias(ours, truth):.2e} cudnn {_bias(ref32, truth):.2e}")
    assert e_ours < 3e-7 and e_ours <= 4 * e_ref + 1e-8
    assert _rel(ours, truth) < 2e-6


@pytest.mark.parametrize("N,H,W,Ca,Cb", CASES)
def test_backward_matches_fp64(N, H, W, Ca, Cb):
    torch.backends.cudnn.allow_tf32 = False
    x, w, dy = _mk(N, H, W, Ca, Cb, seed=1)
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    F.conv2d(xd, wd, padding=1).backward(dy.double())
    x1, w1 = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    conv_tc.conv3x3_tc(x1, w1).backward(dy)
    x2, w2 = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    F.conv2d(x2, w2, padding=1).backward(dy)
    for name, ours, ref32, truth in (("dx", x1.grad, x2.grad, xd.grad), ("dw", w1.grad, w2.grad, wd.grad)):
        e_ours, e_ref = _rms(ours, truth), _rms(ref32, truth)
        print(f"{name} {N}x{H}x{W} {Ca}->{Cb}: rms err ours {e_ours:.3e} cudnn-fp32 {e_ref:.3e} | max ours "
              f"{_rel(ours, truth):.3e} cudnn {_rel(ref32, truth):.3e} | shrink ours {_bias(ours, truth):.2e} "
              f"cudnn {_bias(ref32, truth):.2e}")
        assert e_ours < 5e-7 and e_ours <= 4 * e_ref + 1e-8, name
        assert _rel(ours, truth) < 4e-6, name
    assert w1.grad.stride() == w1.stride()


KINDS = [  # kind, N, H, W, Cin, Cout, kernel, stride, pad
    ("s2", 4, 32, 32, 64, 128, 3, 2, 1),
    ("s2", 4, 16, 16, 128, 256, 3, 2, 1),
    ("s2", 9, 8, 8, 256, 512, 3, 2, 1),       # 4x4 outputs, 9 images: zero-filled tail of the 8-image tile
    ("p2", 4, 32, 32, 64, 128, 1, 2, 0),
    ("p2", 8, 8, 8, 256, 512, 1, 2, 0),
    ("p1", 4, 16, 16, 64, 256, 1, 1, 0),
    ("stem", 8, 32, 32, 3, 64, 3, 1, 1),
]


@pytest.mark.parametrize("kind,N,H,W,Ci,Co,k,st,pd", KINDS)
def test_strided_pointwise_and_stem_match_fp64(kind, N, H, W, Ci, Co, k, st, pd):
    """the other members of the tap-table family: forward, data gradient and weight gradient against fp64"""
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(N, Ci, H, W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Co, Ci, k, k, device="cuda", generator=g) * (2.0 / (k * k * Ci)) ** 0.5).contiguous(
        memory_format=torch.channels_last)
    assert conv_tc.kind_of(x, w, (st, st), (pd, pd), (1, 1), 1) == kind
    need_dx = kind != "stem"
    xd, wd = x.double().requires_grad_(need_dx), w.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, stride=st, padding=pd)
    dy = torch.randn(yd.shape, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    yd.backward(dy.double())
    x1, w1 = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(True)
    y1 = conv_tc.conv2d(x1, w1, None, (st, st), (pd, pd), (1, 1), 1)
    y1.backward(dy)
    x2, w2 = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(True)
    y2 = F.conv2d(x2, w2, stride=st, padding=pd)
    y2.backward(dy)
    trip = [("y", y1, y2, yd.detach()), ("dw", w1.grad, w2.grad, wd.grad)]
    if need_dx:
        trip.append(("dx", x1.grad, x2.grad, xd.grad))
    for name, ours, ref32, truth in trip:
        e_ours, e_ref = _rms(ours, truth), _rms(ref32, truth)
        print(f"{kind} {name} {N}x{H}x{W} {Ci}->{Co}: rms err ours {e_ours:.3e} cudnn-fp32 {e_ref:.3e} | max ours "
              f"{_rel(ours, truth):.3e} cudnn {_rel(ref32, truth):.3e}")
        assert ours.shape == truth.shape, name
        assert e_ours < 5e-7 and e_ours <= 4 * e_ref + 1e-8, name
        assert _rel(ours, truth) < 4e-6, name
    # same memory order as the parameter (strides of size-1 dims are arbitrary)
    assert [s_ for s_, n in zip(w1.grad.stride(), w1.shape) if n > 1] == [s_ for s_, n in zip(w1.stride(), w1.shape) if n > 1]


def test_wgrad_is_bitwise_reproducible():
    x, w, dy = _mk(4, 16, 16, 128, 128, seed=2)
    outs = []
    for _ in range(3):
        w1 = w.clone().requires_grad_(True)
        conv_tc.conv3x3_tc(x, w1).backward(dy)
        outs.append(w1.grad.clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_whole_resnet_runs_on_the_tensor_core_convs_and_is_as_close_to_fp64_as_cudnn():
    """every conv of the reference ResNet (stem, 3x3 s1/s2, 1x1 s2) takes the wgmma path, BN hands the bf16 planes
    over (no split pass between BN and the next conv), and the gradients of the whole network are as close to an fp64
    run of the same model as the gradients of the cuDNN fp32 run are (a 28-conv BN network amplifies round-off, so
    the two fp32 runs are compared against the TRUTH, not against each other)"""
    import copy
    from eventgrad_b200.models.resnet import make_resnet
    from eventgrad_b200.ops import ext
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    m = make_resnet("resnet18").cuda().to(memory_format=torch.channels_last)
    x = torch.randn(32, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), device="cuda")
    m64 = copy.deepcopy(m).double()
    l64 = F.cross_entropy(m64(x.double()), y)
    l64.backward()
    g64 = torch.cat([p.grad.flatten() for p in m64.parameters()])
    res = {}
    for on in (True, False):
        conv_tc.set_enabled(on)
        m.zero_grad(set_to_none=True)
        before = dict(ext().launch_counts())["conv"]
        loss = F.cross_entropy(m(x), y)
        loss.backward()
        n = dict(ext().launch_counts())["conv"] - before
        g = torch.cat([p.grad.flatten() for p in m.parameters()]).double()
        res[on] = (abs(float(loss) - float(l64)), float((g - g64).norm() / g64.norm()), n)
    conv_tc.set_enabled(None)
    print(f"resnet18-ref vs fp64: |dloss| ours {res[True][0]:.2e} cudnn {res[False][0]:.2e}; grad rel err ours "
          f"{res[True][1]:.3e} cudnn {res[False][1]:.3e}; conv-family launches {res[True][2]}")
    assert res[False][2] == 0 and res[True][2] >= 28 * 3          # 28 convs: fprop + dgrad + wgrad (+ prep / splits)
    # plane hand-over: 21 forward and 28 backward split passes are gone (only the parity / stem gathers remain):
    # 28 x (fprop + wgrad + wgrad-reduce + weight prep) + 24 dgrad + 9 extra launches of the three 4-class stride-2
    # dgrads + 4 gathers = 149, plus one reduce launch per K-split forward/dgrad at this small batch
    assert res[True][2] <= 149 + 2 * 28
    assert res[True][0] <= 3 * res[False][0] + 2e-6
    assert res[True][1] <= 2 * res[False][1] + 1e-6


def test_bottleneck_resnet50_takes_the_tensor_core_path():
    """the BottleNeck family (1x1 stride-1 convs up to 2048 channels, 3x3 stride-2 inside the block, 1x1 stride-1 and
    stride-2 down-samplers): every conv on the wgmma kernels, loss and gradients as close to fp64 as cuDNN's"""
    import copy
    from eventgrad_b200.models.resnet import make_resnet
    from eventgrad_b200.ops import ext
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(1)
    m = make_resnet("resnet50", variant="canonical").cuda().to(memory_format=torch.channels_last)
    x = torch.randn(8, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (8,), device="cuda")
    m64 = copy.deepcopy(m).double()
    l64 = F.cross_entropy(m64(x.double()), y)
    l64.backward()
    g64 = torch.cat([p.grad.flatten() for p in m64.parameters()])
    res = {}
    for on in (True, False):
        conv_tc.set_enabled(on)
        m.zero_grad(set_to_none=True)
        before = dict(ext().launch_counts())["conv"]
        loss = F.cross_entropy(m(x), y)
        loss.backward()
        n = dict(ext().launch_counts())["conv"] - before
        g = torch.cat([p.grad.flatten() for p in m.parameters()]).double()
        res[on] = (abs(float(loss) - float(l64)), float((g - g64).norm() / g64.norm()), n)
    conv_tc.set_enabled(None)
    print(f"resnet50 vs fp64: |dloss| ours {res[True][0]:.2e} cudnn {res[False][0]:.2e}; grad rel err ours "
          f"{res[True][1]:.3e} cudnn {res[False][1]:.3e}; conv-family launches {res[True][2]}")
    n_convs = sum(1 for mod in m.modules() if isinstance(mod, torch.nn.Conv2d))
    assert res[False][2] == 0 and res[True][2] >= 3 * n_convs
    assert res[True][0] <= 3 * res[False][0] + 2e-6
    assert res[True][1] <= 2 * res[False][1] + 1e-6
