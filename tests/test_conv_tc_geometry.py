"""The tensor-core convolutions (csrc/conv_tc.cu) at every kind of pixel tile their eligibility admits, against fp64.

conv_tc_supported accepts every output grid that cuts into 128-row (forward / data gradient) and 64-row (weight
gradient) pixel tiles, and every multiple of 64 channels.  A tile is one of three things:
    part-img    bh full rows of one image; H / bh tiles per image, which need not be a power of two (12x32: 3)
    tile=img    exactly one image (4x32, 8x16, 128x1)
    multi-img   bn whole images (2x2: 32, 1x1: 128); when bn does not divide N the last tile has zero-filled images
On top of the tiling, the launcher picks a 64- or 128-wide channel tile, a K-split of the forward, a pixel split of the
weight gradient and a persistent grid, all from the SM count.  The CIFAR ResNet's layers (test_gpu_conv_tc.py) reach
only square power-of-two grids; this file runs one case for every class of launch.

The CPU tests keep the case table honest: a model of the tiling must agree with the extension, every launch class must
have a case, and the elementwise error bound the GPU tests use must reject the indexing errors a kernel can make.

Elementwise bound: |ours - truth| <= 2^-14 * B, where B is the same operation in fp64 on absolute values (conv(|x|, |w|)
for y; its gradients with upstream |dy| for dx and dW).  Rounding stays far below it: the largest ratio over the cases
below was 2^-22.3 on an H100 SXM (700 W), while a dropped 64-channel block, a wrong halo or a neighbouring image leaking
into a tile errs by 2^-5 B or more (test_bound_passes_rounding_and_rejects_indexing_errors).  2^-14 sits in the middle:
the rounding error of a single fp32 sum grows with its length, and a weight gradient sums hundreds of partials.  Where
B is 0 (taps whose whole window is zero padding) the result must be exactly 0.
"""
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

import test_conv_tc_orchestration as orch
from eventgrad_b200.ops import conv_tc, ext

BOUND = 2.0 ** -14

# ------------------------------------------------------------------------------------------------ tiling model
Geometry = namedtuple("Geometry", "mode bh bn tiles tail")


def geometry(N, H, W, rows):
    """How the kernels cut the pixel grid (N, H, W) into tiles of `rows` pixels, or None when it does not tile."""
    if H * W > rows:                                  # part of an image: bh full rows, bh dividing H
        if rows % W or H % (rows // W):
            return None
        bh = rows // W
        return Geometry("part-img", bh, 1, N * (H // bh), False)
    if rows % (H * W):                                # one or more whole images
        return None
    bn = rows // (H * W)
    if bn == 1:
        return Geometry("tile=img", H, 1, N, False)
    return Geometry("multi-img", H, bn, -(-N // bn), N % bn != 0)


def test_tiling_model_matches_the_extension():
    C = ext()
    bad = []
    for N in (1, 2, 3, 5, 8, 37, 67):
        for H in range(1, 129):
            for W in range(1, 129):
                g128, g64 = geometry(N, H, W, 128), geometry(N, H, W, 64)
                if C.conv_tc_supported(N, H, W, 64, 64) != (g128 is not None and g64 is not None):
                    bad.append((N, H, W, "supported"))
                if C.conv_fprop_mtiles(N, H, W) != (0 if g128 is None else g128.tiles):
                    bad.append((N, H, W, "tiles"))
    assert not bad, bad[:20]


# ------------------------------------------------------------------------------------------------ cases
# (H, W) is the OUTPUT grid, the pixel grid the kernels tile; a stride-2 conv reads a 2H x 2W input.  sm: the SM count
# the launcher plans for (132 = H100 SXM; smaller counts give 128-wide tiles and persistent walks on small grids).
Case = namedtuple("Case", "kind N H W Ci Co sm spread", defaults=(False,))
CASES = [
    Case("s1", 2, 64, 64, 64, 64, 132),         # W = 64; uneven weight-gradient pixel splits
    Case("s1", 6, 4, 32, 128, 192, 132),        # forward tile = one image
    Case("s1", 37, 8, 16, 64, 384, 16),         # one image per tile at NT 128, 3 channel tiles, persistent walk
    Case("s1", 5, 12, 32, 192, 128, 132),       # 3 tiles per image; 27 k-blocks in 4 uneven K splits; U = 27
    Case("s1", 2, 96, 4, 64, 128, 132),         # 3 tiles per image, 4-wide rows
    Case("s1", 21, 2, 2, 256, 256, 132),        # 32 images per tile, zero-filled tail
    Case("s1", 67, 1, 1, 512, 512, 132),        # 128 images per tile: every tap but the centre is padding
    Case("s1", 5, 1, 64, 64, 128, 132),         # 1 x 64 strips
    Case("s1", 3, 128, 1, 64, 64, 132),         # 128 x 1 columns: the horizontal taps are padding
    Case("s1", 9, 8, 8, 256, 256, 16),          # multi-image tile with a tail at NT 128
    # 160 work items on 36 CTAs at NT 64.  Planned for fewer SMs, the weight gradient runs un-split: 160 k-blocks in one
    # fp32 sum, whose rms error (5.1e-7 on an H100, cuDNN fp32: 5.1e-6) crosses the absolute 5e-7 cap of the yardstick
    Case("s1", 40, 16, 16, 128, 128, 36),
    Case("s2", 9, 2, 2, 512, 512, 132),         # 4x4 input
    Case("s2", 5, 1, 1, 256, 512, 132),         # 2x2 input
    Case("s2", 3, 12, 32, 64, 128, 132),        # 24x64 input
    Case("p1", 6, 8, 8, 192, 320, 132),         # 5 channel tiles; weight gradient U = 3
    Case("p1", 2, 64, 64, 64, 128, 5),          # NT 128 walk over part-image tiles; U = 1
    Case("p2", 70, 1, 1, 256, 512, 132),        # 2x2 input
    Case("stem", 3, 24, 16, 3, 64, 132),
    Case("stem", 9, 1, 1, 3, 64, 132),
    Case("s1", 4, 16, 16, 128, 128, 132, True),  # x scaled per channel over 12 decades
]


def _cid(c):
    return f"{c.kind}-{c.N}x{c.H}x{c.W}-{c.Ci}to{c.Co}-sm{c.sm}" + ("-spread" if c.spread else "")


def launches(c):
    """(kernel, Ca, Cb, ntaps) of every launch of the forward, data gradient and weight gradient of case c"""
    T = 9 if c.kind in ("s1", "s2") else 1
    Ci = 64 if c.kind == "stem" else c.Ci              # the stem's 27 (tap, rgb) values are one 64-wide K block
    out = [("fprop", Ci, c.Co, T), ("wgrad", Ci, c.Co, T)]
    if c.kind == "s2":                                 # one data-gradient launch per input parity class
        out += [("fprop", c.Co, Ci, len(t)) for t in conv_tc.TAPS_S2_DGRAD.values()]
    elif c.kind != "stem":
        out.append(("fprop", c.Co, Ci, T))
    return out


def _uneven(n, splits):
    """n blocks in `splits` ranges of ceil(n / splits): is the last range shorter?"""
    per = -(-n // splits)
    return splits > 1 and n - (splits - 1) * per != per


def launch_classes(c):
    C = ext()
    N, H, W, sm = c.N, c.H, c.W, c.sm
    got = set()
    for kern, Ca, Cb, T in launches(c):
        g = geometry(N, H, W, 128 if kern == "fprop" else 64)
        tiling = g.mode + ("+tail" if g.tail else "")
        got.add(f"{kern} {tiling}")
        if kern == "fprop":
            NT = C.conv_fprop_ntile(N, H, W, Ca, Cb, T, sm)
            ks = C.conv_fprop_ksplits(N, H, W, Ca, Cb, T, sm)
            if g.mode == "part-img":
                tpi = H // g.bh
                got.add("fprop part-img tpi " + ("2^k" if tpi & (tpi - 1) == 0 else "not 2^k"))
            got.add(f"fprop NT{NT} {tiling}")
            if _uneven(T * Ca // 64, ks):
                got.add("fprop uneven K split")
            if ks == 1 and g.tiles * (Cb // NT) > sm:
                got.add(f"fprop walk NT{NT}")
            if Cb // NT >= 3 and Cb // NT % 2:
                got.add("fprop odd channel tiles >= 3")
        else:
            U, s = T * Ca // 64, C.conv_wgrad_splits(N, H, W, Ca, Cb, T, sm)
            if s == 1:
                got.add("wgrad 1 split")
            if _uneven(g.tiles, s):
                got.add("wgrad uneven splits")
            if U == 1 or U % 2:
                got.add("wgrad U=1" if U == 1 else "wgrad U odd > 1")
    if not (H == W and H in (4, 8, 16, 32)):
        got.add(f"{c.kind} off the square grids")
    got |= {lbl for lbl, on in (("grid 1x1", H == W == 1), ("grid 2x2", H == W == 2), ("W=64", W == 64),
                                 ("H!=W", H != W)) if on}
    return got


REQUIRED = {
    "fprop part-img tpi 2^k", "fprop part-img tpi not 2^k", "fprop tile=img", "fprop multi-img",
    "fprop multi-img+tail",
    "wgrad part-img", "wgrad tile=img", "wgrad multi-img+tail",
    "fprop NT128 part-img", "fprop NT128 tile=img", "fprop NT128 multi-img+tail",
    "fprop uneven K split", "fprop walk NT64", "fprop walk NT128",
    "wgrad 1 split", "wgrad uneven splits", "wgrad U=1", "wgrad U odd > 1",
    "fprop odd channel tiles >= 3",
    "s1 off the square grids", "s2 off the square grids", "p1 off the square grids", "p2 off the square grids",
    "stem off the square grids",
    "grid 1x1", "grid 2x2", "W=64", "H!=W",
}


def test_every_launch_class_has_a_gpu_case():
    """a change to the tiling, the N-tile rule or the split rules that leaves a class without a case fails here"""
    C = ext()
    for c in CASES:
        assert C.conv_tc_supported(c.N, c.H, c.W, 64 if c.kind == "stem" else c.Ci, c.Co), c
    union = set().union(*(launch_classes(c) for c in CASES))
    assert REQUIRED <= union, sorted(REQUIRED - union)


# ------------------------------------------------------------------------------------------------ the bound
def bound_check(ours, truth, B):
    """(max |ours - truth| / B where B > 0, whether ours is exactly 0 wherever B is 0)"""
    ours = ours.detach().double()
    zero = B == 0
    ratio = float(((ours - truth).abs()[~zero] / B[~zero]).max()) if bool((~zero).any()) else 0.0
    return ratio, bool((ours[zero] == 0).all())


def _conv_args(kind):
    return {"s1": (1, 1), "s2": (2, 1), "p1": (1, 0), "p2": (2, 0), "stem": (1, 1)}[kind]


def fp64_truth_and_bound(x, w, dy, stride, pad, need_dx):
    """fp64 (y, dx, dw) of the convolution and the same on absolute values: the elementwise bounds B"""
    res = []
    for xs, ws, gs in ((x, w, dy), (x.abs(), w.abs(), dy.abs())):
        xd = xs.detach().double().requires_grad_(need_dx)
        wd = ws.detach().double().requires_grad_(True)
        y = F.conv2d(xd, wd, stride=stride, padding=pad)
        y.backward(gs.double())
        res.append((y.detach(), xd.grad, wd.grad))
    return res


# ------------------------------------------------------------------------------------------------ CPU: the bound
# separates rounding from indexing errors, on the emulated primitives of the orchestration tests (fp32 arithmetic)
MUTATION_GEOMS = {  # N, H, W, Ci, Co of an s1 conv
    "12x32": (5, 12, 32, 192, 128),            # part-img, 3 tiles per image
    "2x2": (21, 2, 2, 256, 256),               # 32 images per tile, tail
    "1x64": (5, 1, 64, 64, 128),               # 2 images per tile, tail
}


def _emulated_y_dw(x, w, dy, N, H, W, Ci, Co):
    """the s1 forward and weight gradient from the emulated kernel primitives, NCHW / OIHW"""
    xp = orch.emu_split3(x)
    wp, _ = orch.emu_wprep(w.permute(0, 2, 3, 1).reshape(Co, 9, Ci), False)
    y = orch.emu_fprop(xp, wp, N, H, W, Ci, Co, conv_tc.TAPS_S1, 1, 9)
    dw = orch.emu_wgrad(xp, orch.emu_split3(dy), N, H, W, Ci, Co, conv_tc.TAPS_S1, 1)
    return y, dw


def _drop_block(x, w, y, N, H, W, Ci, Co):
    """the second tile (the only one when there is one) misses the last 64-channel block of tap 4 (the centre)"""
    keep = torch.ones(Ci)
    keep[-64:] = 0
    xp_hole = orch.emu_split3((x * keep[None, :, None, None]).contiguous(memory_format=torch.channels_last))
    xp = orch.emu_split3(x)
    wp, _ = orch.emu_wprep(w.permute(0, 2, 3, 1).reshape(Co, 9, Ci), False)
    taps = conv_tc.TAPS_S1
    y_hole = orch.emu_fprop(xp, wp, N, H, W, Ci, Co, taps[:4] + taps[5:], 1, 9) + \
        orch.emu_fprop(xp_hole, wp, N, H, W, Ci, Co, taps[4:5], 1, 9)
    out = y.clone().reshape(-1, Co)
    rows = slice(128, 256) if N * H * W > 128 else slice(0, 128)
    out[rows] = y_hole.reshape(-1, Co)[rows]
    return out.reshape(y.shape)


def _leak_image(y, N, H, W):
    """image 0's rows land in image 1, its neighbour in the first multi-image tile"""
    assert geometry(N, H, W, 128).bn > 1
    out = y.clone()
    out[1] = y[0]
    return out


@pytest.mark.parametrize("geom,mutation", [("12x32", "drop"), ("12x32", "wrap"), ("2x2", "drop"), ("2x2", "leak"),
                                           ("2x2", "wrap"), ("1x64", "drop"), ("1x64", "leak"), ("1x64", "wrap")])
def test_bound_passes_rounding_and_rejects_indexing_errors(monkeypatch, geom, mutation):
    N, H, W, Ci, Co = MUTATION_GEOMS[geom]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(N, Ci, H, W, generator=g).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Co, Ci, 3, 3, generator=g) * (2.0 / (9 * Ci)) ** 0.5).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(N, Co, H, W, generator=g).contiguous(memory_format=torch.channels_last)
    (yt, _, dwt), (yb, _, dwb) = fp64_truth_and_bound(x, w, dy, 1, 1, False)
    y, dw = _emulated_y_dw(x, w, dy, N, H, W, Ci, Co)
    y, dw = y.permute(0, 3, 1, 2), dw.reshape(Co, 3, 3, Ci).permute(0, 3, 1, 2)
    for name, ours, truth, B in (("y", y, yt, yb), ("dw", dw, dwt, dwb)):
        ratio, zeros = bound_check(ours, truth, B)
        assert ratio <= BOUND and zeros, (name, ratio, zeros)
    if mutation == "drop":
        bad = {"y": _drop_block(x, w, y.permute(0, 2, 3, 1), N, H, W, Ci, Co).permute(0, 3, 1, 2)}
    elif mutation == "leak":
        bad = {"y": _leak_image(y, N, H, W)}
    else:                                             # the halo wraps around the image instead of reading zeros
        monkeypatch.setattr(orch, "_shift", lambda a, dh, dw_: torch.roll(a, (-dh, -dw_), dims=(1, 2)))
        ym, dwm = _emulated_y_dw(x, w, dy, N, H, W, Ci, Co)
        bad = {"y": ym.permute(0, 3, 1, 2), "dw": dwm.reshape(Co, 3, 3, Ci).permute(0, 3, 1, 2)}
    for name, ours in bad.items():
        truth, B = (yt, yb) if name == "y" else (dwt, dwb)
        ratio, zeros = bound_check(ours, truth, B)
        print(f"{geom} {mutation} {name}: max |err|/B 2^{math.log2(max(ratio, 1e-300)):.1f}, zeros exact {zeros}")
        assert not (ratio <= BOUND and zeros), (name, ratio)


# ------------------------------------------------------------------------------------------------ GPU
def _rms(a, truth):
    return float(((a.detach().double() - truth) ** 2).mean().sqrt() / (truth ** 2).mean().sqrt())


def _rel(a, truth):
    return float((a.detach().double() - truth).abs().max() / truth.abs().max())


def _patch_sm(monkeypatch, sm):
    dev = torch.device("cuda", torch.cuda.current_device())
    monkeypatch.setitem(conv_tc._SM, dev, min(sm, torch.cuda.get_device_properties(dev).multi_processor_count))


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=_cid)
def test_conv_matches_fp64_elementwise(monkeypatch, c):
    """forward, data gradient (not for the stem) and weight gradient through conv_tc.conv2d against fp64: the rms and
    max yardsticks of test_gpu_conv_tc.py against cuDNN fp32, and the elementwise bound"""
    torch.backends.cudnn.allow_tf32 = False
    _patch_sm(monkeypatch, c.sm)
    st, pd = _conv_args(c.kind)
    k = 1 if c.kind in ("p1", "p2") else 3
    Hin, Win = (c.H * st, c.W * st)
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(c.N, c.Ci, Hin, Win, device="cuda", generator=g)
    if c.spread:
        x = x * torch.logspace(-6, 6, c.Ci, device="cuda")[None, :, None, None]
    x = x.contiguous(memory_format=torch.channels_last)
    w = (torch.randn(c.Co, c.Ci, k, k, device="cuda", generator=g) * (2.0 / (k * k * c.Ci)) ** 0.5).contiguous(
        memory_format=torch.channels_last)
    dy = torch.randn(c.N, c.Co, c.H, c.W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    need_dx = c.kind != "stem"
    (yt, dxt, dwt), (yb, dxb, dwb) = fp64_truth_and_bound(x, w, dy, st, pd, need_dx)
    x1, w1 = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(True)
    assert conv_tc.kind_of(x1, w1, (st, st), (pd, pd), (1, 1), 1) == c.kind
    y1 = conv_tc.conv2d(x1, w1, None, (st, st), (pd, pd), (1, 1), 1)
    y1.backward(dy)
    x2, w2 = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(True)
    y2 = F.conv2d(x2, w2, stride=st, padding=pd)
    y2.backward(dy)
    torch.cuda.synchronize()
    trip = [("y", y1, y2, yt, yb), ("dw", w1.grad, w2.grad, dwt, dwb)]
    if need_dx:
        trip.append(("dx", x1.grad, x2.grad, dxt, dxb))
    fails = []
    for name, ours, ref32, truth, B in trip:
        assert ours.shape == truth.shape, name
        e_ours, e_ref, rel = _rms(ours, truth), _rms(ref32, truth), _rel(ours, truth)
        ratio, zeros = bound_check(ours, truth, B)
        print(f"{_cid(c)} {name}: max |err|/B {ratio:.3e} (2^{math.log2(max(ratio, 1e-300)):.1f}) zeros exact {zeros}"
              f" | rms ours {e_ours:.3e} cudnn-fp32 {e_ref:.3e} | max/max {rel:.3e}")
        if not (e_ours < 5e-7 and e_ours <= 4 * e_ref + 1e-8 and rel < 4e-6 and ratio <= BOUND and zeros):
            fails.append((name, e_ours, e_ref, rel, ratio, zeros))
    assert not fails, fails
    assert [s for s, n in zip(w1.grad.stride(), w1.shape) if n > 1] == [s for s, n in zip(w1.stride(), w1.shape) if n > 1]


SKIP_CASES = [  # N, H, W, Ca, Cb, sm: the s1 data gradient's epilogue adds the masked skip-connection gradient
    (40, 16, 16, 128, 128, 36, 64, 1),         # NT 64, un-split, persistent walk
    (9, 8, 8, 256, 256, 16, 128, 1),           # NT 128, un-split, multi-image tiles with a tail
    (5, 12, 32, 192, 128, 132, 64, 4),         # K split: the reduce kernel adds it
]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Ca,Cb,sm,NT,ks", SKIP_CASES)
def test_skip_gradient_epilogue_matches_fp64(monkeypatch, N, H, W, Ca, Cb, sm, NT, ks):
    """fprop(..., addend, addmask) = conv + (mask bit ? addend : 0), the mask bit of flat NHWC index off being bit
    off & 7 of byte off >> 3"""
    _patch_sm(monkeypatch, sm)
    C = ext()
    assert (C.conv_fprop_ntile(N, H, W, Ca, Cb, 9, sm), C.conv_fprop_ksplits(N, H, W, Ca, Cb, 9, sm)) == (NT, ks)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(N, Ca, H, W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Cb, Ca, 3, 3, device="cuda", generator=g) * (2.0 / (9 * Ca)) ** 0.5).contiguous(
        memory_format=torch.channels_last)
    addend = torch.randn(N, H, W, Cb, device="cuda", generator=g)
    mask = torch.randint(0, 256, ((addend.numel() + 7) // 8,), device="cuda", generator=g, dtype=torch.uint8)
    wp, _ = conv_tc.wprep(w.permute(0, 2, 3, 1).reshape(Cb, 9, Ca), False)
    ours = conv_tc.fprop(conv_tc.split3(x), wp, N, H, W, Ca, Cb, conv_tc.TAPS_S1, 1, 9, addend=addend, addmask=mask)
    off = torch.arange(addend.numel(), device="cuda")
    bit = ((mask.long()[off >> 3] >> (off & 7)) & 1).bool().reshape(addend.shape)
    truth = F.conv2d(x.double(), w.double(), padding=1).permute(0, 2, 3, 1)
    B = F.conv2d(x.double().abs(), w.double().abs(), padding=1).permute(0, 2, 3, 1)
    ref = truth + torch.where(bit, addend.double(), 0.0)
    err = (ours.double() - ref).abs()
    worst = float((err / (BOUND * B + 2.0 ** -24 * ref.abs())).max())
    print(f"skip-gradient {N}x{H}x{W} {Ca}->{Cb} sm {sm} NT {NT} ks {ks}: max |err| / bound {worst:.3e}, "
          f"{int(bit.sum())} of {bit.numel()} added")
    assert worst <= 1.0
