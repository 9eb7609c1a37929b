"""CPU check of the N-tile choice of the forward / data-gradient convolution kernel (csrc/conv_tc.cu,
conv_fprop_ntile): 128 output channels only where the 128-wide grid keeps the GPU as busy as the 64-wide one."""
from eventgrad_b200.ops import ext

SMS = 132   # H100 SXM


def test_batch_256_layers_take_the_wide_tile():
    C = ext()
    assert C.conv_fprop_ntile(256, 16, 16, 128, 128, 9, SMS) == 128     # 512 tiles of 128 x 128
    assert C.conv_fprop_ntile(256, 8, 8, 256, 256, 9, SMS) == 128       # 256
    assert C.conv_fprop_ntile(256, 4, 4, 512, 512, 9, SMS) == 128       # 128 tiles: one wave, 256 at 64 wide: two
    assert C.conv_fprop_ntile(256, 16, 16, 64, 128, 9, SMS) == 128      # stride-2 conv into layer 2 (parity grid)
    assert C.conv_fprop_ntile(256, 8, 8, 256, 128, 4, SMS) == 128       # its data gradient, one parity class


def test_64_channel_outputs_keep_the_narrow_tile():
    C = ext()
    assert C.conv_fprop_ntile(256, 32, 32, 64, 64, 9, SMS) == 64
    assert C.conv_fprop_ntile(256, 16, 16, 128, 64, 4, SMS) == 64       # data gradient into a 64-channel input


def test_small_grids_keep_the_narrow_tile():
    C = ext()
    # un-split, but the 128-wide grid would fill only half the SMs (the per-GPU batches of 2-8 GPUs)
    assert C.conv_fprop_ksplits(32, 16, 16, 128, 128, 9, SMS) == 1
    assert C.conv_fprop_ntile(32, 16, 16, 128, 128, 9, SMS) == 64       # 64 tiles at 128 wide, 128 at 64 wide
    assert C.conv_fprop_ntile(64, 8, 8, 256, 256, 9, SMS) == 64
    assert C.conv_fprop_ntile(128, 4, 4, 512, 512, 9, SMS) == 64
    assert C.conv_fprop_ksplits(32, 8, 8, 128, 256, 1, SMS) == 1        # 1x1: not split only because K is 2 blocks
    assert C.conv_fprop_ntile(32, 8, 8, 128, 256, 1, SMS) == 64
    # K-split launches always run 64 wide
    assert C.conv_fprop_ksplits(32, 4, 4, 512, 512, 9, SMS) == 4
    assert C.conv_fprop_ntile(32, 4, 4, 512, 512, 9, SMS) == 64
    # 67..132 tiles of 128: one wave either way
    assert C.conv_fprop_ntile(40, 16, 16, 128, 128, 9, SMS) == 128
    # 140 tiles of 128: two waves of twice the work against three waves at 64 wide
    assert C.conv_fprop_ntile(70, 16, 16, 128, 128, 9, SMS) == 64
