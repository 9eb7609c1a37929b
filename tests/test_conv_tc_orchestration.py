"""CPU oracle for the host side of the tensor-core convolutions (ops/conv_tc.py).

The CUDA primitives (split3*, wprep, fprop, wgrad -- csrc/conv_tc.cu) are replaced by plain PyTorch implementations of
their documented semantics: planes that sum to the fp32 value, the tap table (dh, dw, source sub-image, weight slice),
zero fill outside the image, the strided output scatter.  With those in place the REAL autograd Function
(_ConvTcFn: which planes, which tap tables, which weight layouts, four-class stride-2 data gradient, stem gather, ...) must
reproduce F.conv2d's forward and both gradients for every kind of convolution.  The kernels themselves are checked
against fp64 on a GPU in tests/test_gpu_conv_tc.py; this file keeps the orchestration honest without one.
"""
import pytest
import torch
import torch.nn.functional as F

from eventgrad_b200.ops import conv_tc as ct


def _planes(x):
    a = x.to(torch.bfloat16)
    r1 = x - a.float()
    b = r1.to(torch.bfloat16)
    c = (r1 - b.float()).to(torch.bfloat16)
    return torch.stack([a.flatten(), b.flatten(), c.flatten()])


def _unplanes(p, shape):
    return (p[2].float() + p[1].float() + p[0].float()).reshape(shape)


def emu_split3(x):
    # same MEMORY order as the tensor (channels_last tensors are NHWC in memory)
    if x.dim() == 4 and x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous():
        x = x.permute(0, 2, 3, 1)
    return _planes(x.contiguous())


def emu_split3_parity(x_nhwc):
    N, H, W, C = x_nhwc.shape
    subs = torch.stack([x_nhwc[:, p::2, q::2, :] for p in (0, 1) for q in (0, 1)])       # [4,N,H/2,W/2,C]
    return _planes(subs.contiguous()).reshape(3, 4, N, H // 2, W // 2, C)


def emu_split3_stem(x_nhwc):
    N, H, W, C = x_nhwc.shape
    xp = F.pad(x_nhwc, (0, 0, 1, 1, 1, 1))
    out = torch.zeros(N, H, W, 64)
    for r in range(3):
        for s in range(3):
            out[..., (r * 3 + s) * 3:(r * 3 + s) * 3 + 3] = xp[:, r:r + H, s:s + W, :]
    return _planes(out).reshape(3, N, H, W, 64)


def emu_wprep(w_oti, transposed):
    Co, T, Ci = w_oti.shape
    wp = _planes(w_oti.contiguous()).reshape(3, Co, T * Ci)
    wtp = _planes(w_oti.permute(2, 1, 0).contiguous()).reshape(3, Ci, T * Co) if transposed else None
    return wp, wtp


def _shift(a, dh, dw):
    """a [N,H,W,C] -> b[n,i,j] = a[n,i+dh,j+dw] with zeros outside"""
    N, H, W, C = a.shape
    b = torch.zeros_like(a)
    i0, i1 = max(0, -dh), min(H, H - dh)
    j0, j1 = max(0, -dw), min(W, W - dw)
    if i1 > i0 and j1 > j0:
        b[:, i0:i1, j0:j1] = a[:, i0 + dh:i1 + dh, j0 + dw:j1 + dw]
    return b


def emu_fprop(ap, wp, N, H, W, Ca, Cb, taps, nsrc=1, wtaps=9, out=None, OH=None, OW=None, os_=1, op=0, oq=0):
    OH, OW = OH or H, OW or W
    A = _unplanes(ap.reshape(3, -1), (nsrc, N, H, W, Ca))
    Wt = _unplanes(wp.reshape(3, -1), (Cb, wtaps, Ca))
    if out is None:
        out = torch.empty(N, OH, OW, Cb)
    acc = torch.zeros(N, H, W, Cb)
    for (dh, dw, src, wk) in taps:
        acc += _shift(A[src], dh, dw) @ Wt[:, wk, :].t()
    out[:, op::os_, oq::os_, :][:, :H, :W] = acc
    return out


def emu_wgrad(xp, gp, N, H, W, Ca, Cb, taps, nsrc=1):
    X = _unplanes(xp.reshape(3, -1), (nsrc, N, H, W, Ca))
    G = _unplanes(gp.reshape(3, -1), (N, H, W, Cb)).reshape(-1, Cb)
    dw = torch.empty(Cb, len(taps), Ca)
    for t, (dh, dw_, src, wk) in enumerate(taps):
        dw[:, t, :] = G.t() @ _shift(X[src], dh, dw_).reshape(-1, Ca)
    return dw


@pytest.fixture
def emulated(monkeypatch):
    for name, fn in (("split3", emu_split3), ("split3_parity", emu_split3_parity), ("split3_stem", emu_split3_stem),
                     ("wprep", emu_wprep), ("fprop", emu_fprop), ("wgrad", emu_wgrad)):
        monkeypatch.setattr(ct, name, fn)
    ct._PARITY_CACHE.update({"ref": None, "ver": -1, "planes": None})
    yield
    ct._PARITY_CACHE.update({"ref": None, "ver": -1, "planes": None})


KINDS = [  # kind, N, H, W, Cin, Cout, k, stride, pad
    ("s1", 2, 8, 8, 8, 16, 3, 1, 1),
    ("s2", 2, 8, 8, 8, 16, 3, 2, 1),
    ("p2", 2, 8, 8, 8, 16, 1, 2, 0),
    ("p1", 2, 4, 4, 8, 16, 1, 1, 0),
    ("stem", 2, 8, 8, 3, 16, 3, 1, 1),
    # grids off the square power-of-two ones (see test_conv_tc_geometry.py): 1x1 images, strips, columns, 3 tiles
    # per image, stride-2 convs on 2x2 / 4x4 / 24x64 inputs
    ("s1", 3, 1, 1, 8, 16, 3, 1, 1),
    ("s1", 2, 1, 64, 8, 16, 3, 1, 1),
    ("s1", 2, 128, 1, 8, 8, 3, 1, 1),
    ("s1", 2, 12, 32, 8, 16, 3, 1, 1),
    ("s2", 5, 2, 2, 8, 16, 3, 2, 1),
    ("s2", 2, 4, 4, 8, 16, 3, 2, 1),
    ("s2", 3, 24, 64, 8, 16, 3, 2, 1),
    ("p2", 7, 2, 2, 8, 16, 1, 2, 0),
    ("p2", 2, 24, 64, 8, 8, 1, 2, 0),
    ("p1", 3, 6, 64, 8, 16, 1, 1, 0),
    ("stem", 3, 1, 1, 3, 16, 3, 1, 1),
    ("stem", 2, 24, 16, 3, 16, 3, 1, 1),
]


@pytest.mark.parametrize("kind,N,H,W,Ci,Co,k,st,pd", KINDS)
def test_autograd_function_reproduces_conv2d(emulated, kind, N, H, W, Ci, Co, k, st, pd):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, Ci, H, W, generator=g).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Co, Ci, k, k, generator=g) * 0.2).contiguous(memory_format=torch.channels_last)
    need_dx = kind != "stem"
    x1, w1 = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(True)
    y1 = ct._ConvTcFn.apply(x1, w1, kind)
    x2, w2 = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(True)
    y2 = F.conv2d(x2, w2, stride=st, padding=pd)
    assert y1.shape == y2.shape
    gy = torch.randn(y2.shape, generator=g).contiguous(memory_format=torch.channels_last)
    y1.backward(gy)
    y2.backward(gy)
    assert torch.allclose(y1, y2, atol=2e-5, rtol=1e-5)
    assert w1.grad.shape == w2.grad.shape and torch.allclose(w1.grad, w2.grad, atol=2e-5, rtol=1e-5)
    if need_dx:
        assert torch.allclose(x1.grad, x2.grad, atol=2e-5, rtol=1e-5)
    # the weight gradient comes back in the parameter's memory order (OHWI for channels_last weights)
    assert [s for s, n in zip(w1.grad.stride(), w1.shape) if n > 1] == [s for s, n in zip(w1.stride(), w1.shape) if n > 1]


def test_downsampling_block_splits_its_input_once(emulated, monkeypatch):
    """the 3x3/stride-2 conv and the 1x1/stride-2 down-sampler of a block read the SAME tensor: one parity split"""
    calls = []
    monkeypatch.setattr(ct, "split3_parity", lambda x: (calls.append(1), emu_split3_parity(x))[1])
    x = torch.randn(2, 8, 8, 8).contiguous(memory_format=torch.channels_last)
    w3 = torch.randn(16, 8, 3, 3).contiguous(memory_format=torch.channels_last)
    w1 = torch.randn(16, 8, 1, 1).contiguous(memory_format=torch.channels_last)
    a = ct._ConvTcFn.apply(x, w3, "s2")
    b = ct._ConvTcFn.apply(x, w1, "p2")
    assert len(calls) == 1
    assert torch.allclose(a, F.conv2d(x, w3, stride=2, padding=1), atol=2e-5)
    assert torch.allclose(b, F.conv2d(x, w1, stride=2), atol=2e-5)
    y = torch.randn_like(x)                                   # another tensor: a fresh split
    ct._ConvTcFn.apply(y, w3, "s2")
    assert len(calls) == 2


def test_planes_handed_over_by_the_producer_are_used_instead_of_a_split(emulated, monkeypatch):
    calls = []
    monkeypatch.setattr(ct, "split3", lambda x: (calls.append(tuple(x.shape)), emu_split3(x))[1])
    x = torch.randn(2, 8, 4, 4).contiguous(memory_format=torch.channels_last)
    w = torch.randn(8, 8, 3, 3).contiguous(memory_format=torch.channels_last)
    ct.planes_put(x, emu_split3(x))                           # what the fused BN kernel does for its output
    y = ct._ConvTcFn.apply(x, w, "s1")
    assert calls == []                                        # the activation was not split again
    assert torch.allclose(y, F.conv2d(x, w, padding=1), atol=2e-5)
