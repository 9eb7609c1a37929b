"""CPU checks behind csrc/conv_tc.cu: the 3 x bf16 split and the six-term product really reach fp32 accuracy, and the
host-side tile geometry accepts exactly the shapes the kernels can tile.  (The kernels themselves are tested on a
GPU in tests/test_gpu_conv_tc.py.)"""
import torch
import torch.nn.functional as F

from eventgrad_b200.ops import ext


def split3_ref(x):
    a = x.to(torch.bfloat16).float()
    r1 = x - a
    b = r1.to(torch.bfloat16).float()
    r2 = r1 - b
    c = r2.to(torch.bfloat16).float()
    return a, b, c


def test_three_bf16_planes_carry_24_bits():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1 << 16, generator=g) * torch.logspace(-8, 8, 1 << 16)
    a, b, c = split3_ref(x)
    back = a.double() + b.double() + c.double()
    rel = ((back - x.double()).abs() / x.double().abs()).max()
    assert float(rel) <= 2.0 ** -23


def test_six_term_product_is_as_accurate_as_fp32():
    """conv as six bf16 x bf16 convolutions accumulated in fp32 (what the tensor cores compute) vs plain fp32, both
    against fp64."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 64, 8, 8, generator=g)
    w = torch.randn(64, 64, 3, 3, generator=g) * (2.0 / 576) ** 0.5
    truth = F.conv2d(x.double(), w.double(), padding=1)
    xs, ws = split3_ref(x), split3_ref(w)
    acc = torch.zeros_like(truth, dtype=torch.float32)
    for i, j in ((2, 0), (0, 2), (1, 1), (1, 0), (0, 1), (0, 0)):      # the kernel's order: small terms first
        acc = acc + F.conv2d(xs[i], ws[j], padding=1)
    ref32 = F.conv2d(x, w, padding=1)

    def rms(a):
        return float(((a.double() - truth) ** 2).mean().sqrt() / (truth ** 2).mean().sqrt())
    assert rms(acc) < 2e-7
    assert rms(acc) <= 3 * rms(ref32) + 1e-8
    # dropping the second-order terms would NOT be fp32: bf16 x bf16 alone is ~3 decimal digits
    assert rms(F.conv2d(xs[0], ws[0], padding=1)) > 1e-3


def test_tile_geometry():
    C = ext()
    ok = [(256, 32, 32, 64, 64), (32, 32, 32, 64, 64), (256, 16, 16, 128, 128), (256, 8, 8, 256, 256),
          (256, 4, 4, 512, 512), (5, 4, 4, 128, 64), (3, 8, 8, 64, 128), (1, 64, 64, 64, 64)]
    bad = [(8, 32, 32, 3, 64),      # stem: 3 input channels
           (8, 32, 32, 64, 96),     # Cout not a multiple of 64
           (8, 28, 28, 64, 64),     # width does not divide a 128-pixel tile
           (8, 6, 8, 64, 64)]       # 8x6 images: no whole-image tiling
    for s in ok:
        assert C.conv_tc_supported(*s), s
    for s in bad:
        assert not C.conv_tc_supported(*s), s
    # wgrad splits: enough CTAs to fill the GPU, never more splits than 64-pixel K blocks
    assert C.conv_wgrad_splits(256, 32, 32, 64, 64, 9, 132) == 132 // 5
    assert C.conv_wgrad_splits(256, 4, 4, 512, 512, 9, 132) == 1
    assert C.conv_wgrad_splits(1, 8, 8, 64, 64, 9, 132) == 1
    assert C.conv_wgrad_splits(256, 32, 32, 64, 64, 1, 132) == 132      # stem / 1x1: one unit pair


def test_fprop_k_splits_only_for_small_grids():
    C = ext()
    assert C.conv_fprop_ksplits(256, 32, 32, 64, 64, 9, 132) == 1          # 2048 tiles: no split
    assert C.conv_fprop_ksplits(256, 4, 4, 512, 512, 9, 132) == 1          # 256 tiles
    ks = C.conv_fprop_ksplits(32, 4, 4, 512, 512, 9, 132)                  # 32 tiles, 72 k-blocks -> 4 splits of 18
    assert ks == 4 and C.conv_fprop_mtiles(32, 4, 4) == 4
    ks = C.conv_fprop_ksplits(32, 8, 8, 256, 256, 9, 132)                  # 64 tiles, 36 k-blocks -> 2 splits of 18
    assert ks == 2
    assert C.conv_fprop_ksplits(32, 16, 16, 64, 128, 1, 132) == 1          # 1x1 with one k-block: nothing to split


def test_tap_tables():
    """the tap tables of ops/conv_tc.py against the definition of the strided convolution and its transpose"""
    from eventgrad_b200.ops import conv_tc as ct
    # forward stride 2 / pad 1: output row ho reads input row 2*ho + r - 1 = 2*(ho + dh) + parity
    for (dh, dw, src, wk) in ct.TAPS_S2:
        r, s = divmod(wk, 3)
        ph, pw = divmod(src, 2)
        assert 2 * dh + ph == r - 1 and 2 * dw + pw == s - 1
    # data gradient: input row 2*i + p receives from output row i + a through filter row r  <=>  2*(i+a) + r - 1 == 2*i + p
    seen = set()
    for (p, q), taps in ct.TAPS_S2_DGRAD.items():
        for (a, b, src, wk) in taps:
            r, s = divmod(wk, 3)
            assert src == 0 and 2 * a + r - 1 == p and 2 * b + s - 1 == q
            seen.add(wk)
    assert seen == set(range(9)) and sum(len(t) for t in ct.TAPS_S2_DGRAD.values()) == 9
    assert [t[3] for t in ct.TAPS_S1_DGRAD] == list(range(8, -1, -1))


def test_s2_dgrad_by_parity_classes_matches_autograd():
    """emulate the four-launch data gradient of the stride-2 conv with plain tensor ops"""
    from eventgrad_b200.ops import conv_tc as ct
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(5, 4, 3, 3, generator=g, dtype=torch.float64)
    dy = torch.randn(2, 5, 4, 4, generator=g, dtype=torch.float64)
    F.conv2d(x, w, stride=2, padding=1).backward(dy)
    dx = torch.zeros(2, 4, 8, 8, dtype=torch.float64)
    dyp = F.pad(dy, (1, 1, 1, 1))                      # zero outside, like the TMA fill
    for (p, q), taps in ct.TAPS_S2_DGRAD.items():
        acc = torch.zeros(2, 4, 4, 4, dtype=torch.float64)
        for (a, b, _, wk) in taps:
            r, s = divmod(wk, 3)
            win = dyp[:, :, 1 + a:5 + a, 1 + b:5 + b]                  # dY[i + a, j + b]
            acc += torch.einsum("nohw,oc->nchw", win, w[:, :, r, s])
        dx[:, :, p::2, q::2] = acc
    assert torch.allclose(dx, x.grad, atol=1e-12)


def test_s2_forward_by_parity_images_matches_conv():
    from eventgrad_b200.ops import conv_tc as ct
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    w = torch.randn(5, 4, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, stride=2, padding=1)
    y = torch.zeros_like(ref)
    for (dh, dw, src, wk) in ct.TAPS_S2:
        r, s = divmod(wk, 3)
        ph, pw = divmod(src, 2)
        sub = F.pad(x[:, :, ph::2, pw::2], (1, 1, 1, 1))               # parity image, zero outside
        win = sub[:, :, 1 + dh:5 + dh, 1 + dw:5 + dw]
        y += torch.einsum("nchw,oc->nohw", win, w[:, :, r, s])
    assert torch.allclose(y, ref, atol=1e-12)


def test_cpu_and_ineligible_shapes_fall_back_to_library_conv():
    from eventgrad_b200.ops import conv_tc
    x = torch.randn(2, 64, 8, 8)
    w = torch.randn(64, 64, 3, 3)
    assert not conv_tc.eligible(x, w, (1, 1), (1, 1), (1, 1), 1)
    assert torch.equal(conv_tc.conv2d(x, w, None, (1, 1), (1, 1), (1, 1), 1), F.conv2d(x, w, padding=1))


def test_plane_registry_matches_by_identity_and_version_and_dies_with_the_tensor():
    """ops/conv_tc.py hand-over of bf16 planes from the BN kernels to the convs (CPU tensors suffice for the logic)"""
    import gc
    from eventgrad_b200.ops import conv_tc as ct
    t = torch.zeros(4, 8)
    planes = torch.zeros(3, t.numel(), dtype=torch.bfloat16)
    ct.planes_put(t, planes)
    assert ct.planes_get(t) is planes
    alias = t.view(4, 8)                       # same memory, another tensor object: not a match
    assert ct.planes_get(alias) is None
    t.add_(1)                                  # in-place change: the planes are stale
    assert ct.planes_get(t) is None
    ct.planes_put(t, planes)
    key = t.data_ptr()
    assert key in ct._PLANES
    del t, alias
    gc.collect()
    assert key not in ct._PLANES               # entry removed by the weakref callback
    wrong = torch.zeros(2, 8)
    ct.planes_put(wrong, planes)               # planes of another size are never handed out
    assert ct.planes_get(wrong) is None
