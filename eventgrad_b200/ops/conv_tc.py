"""Convolutions on the wgmma tensor cores at fp32 accuracy: front-end of csrc/conv_tc.cu.

The reference's convolutions are fp32 (/root/reference/dcifar10/common/resnet.hpp:3-9, event.cpp:259-276).  fp32 has
no tensor-core path in cuDNN (SIMT kernels, 67 TFLOP/s peak on an H100 SXM), so the forward, the data gradient and the weight
gradient of every convolution of the ResNet family run here instead: each fp32 tensor is split into three bf16 planes
(x = x0+x1+x2, 24 mantissa bits) and every product is rebuilt from six bf16 tensor-core MMAs accumulated in fp32 --
fp32 storage, fp32 accuracy (measured against fp64 in tests/test_gpu_conv_tc.py on an H100: 0.6-1.7e-7 rms, below
cuDNN's fp32 kernels in every layer shape), tensor-core throughput.

One kernel pair + a tap table (dh, dw, source sub-image, weight slice) serves five kinds of convolution:
    s1    3x3 stride 1 pad 1                     (BasicBlock / BottleNeck body)
    s2    3x3 stride 2 pad 1                     (first conv of a down-sampling block) -- the input is split into its
                                                 four (h%2, w%2) parity images, so every tap is a unit-stride box
    p2    1x1 stride 2 pad 0                     (the down-sampler), p1: 1x1 stride 1 (BottleNeck)
    stem  3x3 stride 1 pad 1 with 3 input channels: the 27 (tap, rgb) values are gathered into one 64-wide K block
Eligibility: CUDA, fp32, channels_last activations, no bias / dilation / groups, channel counts multiples of 64
(stem: Cin = 3), pixel grids that tile (see conv_tc_supported); anything else falls back to F.conv2d (cuDNN).
"""
from __future__ import annotations

import os
import weakref

import torch
import torch.nn.functional as F

_SM = {}


def _sm(device) -> int:
    n = _SM.get(device)
    if n is None:
        n = _SM[device] = torch.cuda.get_device_properties(device).multi_processor_count
    return n


_FORCE = {"on": None}


def set_enabled(on) -> None:
    """Trainer switch (TrainConfig.conv_tc): True / False, or None = follow EGB_CONV_TC (default on)."""
    _FORCE["on"] = on


def enabled() -> bool:
    if _FORCE["on"] is not None:
        return bool(_FORCE["on"])
    return os.environ.get("EGB_CONV_TC", "1") != "0"


# ------------------------------------------------------------------------------------------------ plane registry
# The fused BN kernels (ops/bn_act.py) can emit their output ALSO as three bf16 planes: the activation that feeds the
# next conv (forward) and the gradient that feeds the previous conv's backward.  They are handed over here, keyed by
# the tensor's address and validated by object identity + version, so a conv that finds its operand already split
# skips the split pass.  Entries die with the tensor (weakref callback); a miss is only a missed optimisation.
_PLANES = {}


def planes_put(t: torch.Tensor, planes: torch.Tensor) -> None:
    import weakref
    key = t.data_ptr()

    def _gone(r, k=key):
        e = _PLANES.get(k)
        if e is not None and e[0] is r:
            _PLANES.pop(k, None)
    _PLANES[key] = (weakref.ref(t, _gone), t._version, planes)


def planes_get(t: torch.Tensor):
    e = _PLANES.get(t.data_ptr())
    if e is not None and e[0]() is t and e[1] == t._version and e[2].numel() == 3 * t.numel():
        return e[2]
    return None


def mark_tc_output(y: torch.Tensor) -> torch.Tensor:
    """tag a conv output produced here: the BN that consumes it emits the planes of its input gradient"""
    y._egb_tc = True
    return y


# ------------------------------------------------------------------------------------------------ tap tables
# (dh, dw, source sub-image, weight slice).  Weight slices index the OHWI weight's tap axis (r*3 + s).
TAPS_S1 = [(r - 1, s - 1, 0, r * 3 + s) for r in range(3) for s in range(3)]
# dX[p] = sum_t' dY[p + off(t')] W[.., 8 - t', ..]: same windows, mirrored weight slice of the transposed weights
TAPS_S1_DGRAD = [(r - 1, s - 1, 0, 8 - (r * 3 + s)) for r in range(3) for s in range(3)]
TAPS_1X1 = [(0, 0, 0, 0)]


def _par(r):
    """input row 2*ho + r - 1 of a stride-2 / pad-1 conv -> (parity image, shift inside it)"""
    return {0: (1, -1), 1: (0, 0), 2: (1, 0)}[r]


TAPS_S2 = [(_par(r)[1], _par(s)[1], _par(r)[0] * 2 + _par(s)[0], r * 3 + s) for r in range(3) for s in range(3)]
# data gradient of the stride-2 conv, one launch per INPUT parity class (p, q): input row 2i+p receives from output
# row i + a through filter row r, for (r, a) in _DG[p]
_DG = {0: [(1, 0)], 1: [(0, 1), (2, 0)]}
TAPS_S2_DGRAD = {(p, q): [(a, b, 0, r * 3 + s) for (r, a) in _DG[p] for (s, b) in _DG[q]] for p in (0, 1) for q in (0, 1)}


# ------------------------------------------------------------------------------------------------ raw kernel calls
def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def split3(x: torch.Tensor) -> torch.Tensor:
    """fp32 tensor (dense in memory, any dim order) -> bf16 planes [3, numel] in the SAME memory order."""
    from . import ext
    n = x.numel()
    assert x.dtype == torch.float32 and n % 8 == 0
    out = torch.empty(3, n, dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device):
        ext().split3(x.data_ptr(), out.data_ptr(), n, _stream(x.device))
    return out


def split3_parity(x_nhwc: torch.Tensor) -> torch.Tensor:
    """[N,H,W,C] fp32 -> planes [3,4,N,H/2,W/2,C]: the four parity images of a stride-2 conv's input."""
    from . import ext
    N, H, W, C = x_nhwc.shape
    out = torch.empty(3, 4, N, H // 2, W // 2, C, dtype=torch.bfloat16, device=x_nhwc.device)
    with torch.cuda.device(x_nhwc.device):
        ext().split3_parity(x_nhwc.data_ptr(), out.data_ptr(), N, H, W, C, _stream(x_nhwc.device))
    return out


def split3_stem(x_nhwc: torch.Tensor) -> torch.Tensor:
    """[N,H,W,3] fp32 -> planes [3,N,H,W,64]: channel k = (r*3+s)*3 + c of pixel (h,w) is x[h+r-1, w+s-1, c]."""
    from . import ext
    N, H, W, C = x_nhwc.shape
    assert C == 3
    out = torch.empty(3, N, H, W, 64, dtype=torch.bfloat16, device=x_nhwc.device)
    with torch.cuda.device(x_nhwc.device):
        ext().split3_stem(x_nhwc.data_ptr(), out.data_ptr(), N, H, W, _stream(x_nhwc.device))
    return out


def wprep(w_oti: torch.Tensor, transposed: bool):
    """fp32 [Co,T,Ci] -> (planes [3,Co,T*Ci], planes [3,Ci,T*Co] or None)"""
    from . import ext
    Co, T, Ci = w_oti.shape
    wp = torch.empty(3, Co, T * Ci, dtype=torch.bfloat16, device=w_oti.device)
    wtp = torch.empty(3, Ci, T * Co, dtype=torch.bfloat16, device=w_oti.device) if transposed else None
    with torch.cuda.device(w_oti.device):
        ext().conv_wprep(w_oti.data_ptr(), wp.data_ptr(), 0 if wtp is None else wtp.data_ptr(), Co, T, Ci,
                         _stream(w_oti.device))
    return wp, wtp


KSPLIT = os.environ.get("EGB_CONV_KSPLIT", "1") != "0"
# weight gradient on a side stream, concurrent with the data gradient of the same layer and, when the join can wait for
# the end of the backward (_fork_wgrad.join), with the layers after it (branches inside the step's CUDA graph)
PAR_BWD = os.environ.get("EGB_CONV_PAR_BWD", "1") != "0"
_SIDE = {}


class _fork_wgrad:
    """context: run the enclosed launches on the side stream, ordered after everything enqueued so far on the current
    stream; `join()` makes the current stream wait for them"""

    def __init__(self, dev, on):
        self.on = on = bool(on) and torch.device(dev).type == "cuda"
        if on:
            self.cur = torch.cuda.current_stream(dev)
            self.side = _SIDE.get(dev)
            if self.side is None:
                self.side = _SIDE[dev] = torch.cuda.Stream(dev)
            self.ctx = torch.cuda.stream(self.side)

    def __enter__(self):
        if self.on:
            self.side.wait_stream(self.cur)
            self.ctx.__enter__()
        return self

    def __exit__(self, *a):
        if self.on:
            self.ctx.__exit__(*a)
        return False

    def join(self, dw, weight, *read):
        """Order the wgrad's result `dw` before its readers.  When the only reader is the AccumulateGrad of a leaf
        weight without a preset .grad (it steals dw as the new .grad, no kernel), the wait is deferred to the end of
        the backward pass (`_join_at_end`), so the side stream keeps running under the following layers' work.
        Otherwise (preset .grad: AccumulateGrad adds dw in place; hooks; a non-leaf weight; outside a backward pass)
        the current stream waits here.  `read`: the tensors the wgrad reads, kept alive for the side stream (dw and
        the split workspace were allocated on the side stream, which orders their reuse there)."""
        if not self.on:
            return
        dw.record_stream(self.cur)
        if _defer_ok(dw, weight):
            for t in read:
                t.record_stream(self.side)
            _join_at_end(self.cur, self.side)
        else:
            self.cur.wait_stream(self.side)


def _defer_ok(dw, w) -> bool:
    return (w is not None and w.is_leaf and w.requires_grad and w.grad is None and not w._backward_hooks
            and not getattr(w, "_post_accumulate_grad_hooks", None) and dw.stride() == w.stride()
            and torch._C._current_graph_task_id() != -1)


# backward pass (autograd graph task id) -> {(current stream, side stream)} still to be joined at its end
_PENDING = {}


def _join_at_end(cur, side) -> None:
    """Make `cur` wait for `side` when the running backward pass ends: from a callback of the autograd engine, which
    runs before backward() / autograd.grad() return, so every caller sees the gradients ordered on `cur` (and a
    CUDA-graph capture records the wait, joining the side stream back into the capture)."""
    task = torch._C._current_graph_task_id()
    pend = _PENDING.get(task)
    if pend is None:
        pend = _PENDING[task] = set()

        def _join():
            for c, s in _PENDING.pop(task, ()):
                c.wait_stream(s)
        torch.autograd.Variable._execution_engine.queue_callback(_join)
    pend.add((cur, side))


def fprop(ap, wp, N, H, W, Ca, Cb, taps, nsrc=1, wtaps=9, out=None, OH=None, OW=None, os_=1, op=0, oq=0,
          addend=None, addmask=None):
    """implicit GEMM over the pixel grid (N,H,W): out[n, i*os+op, j*os+oq, :] = sum_taps A_tap[n,i,j,:] @ W_tap^T
    (+ (addmask bit ? addend : 0) when given: fp32 in out's layout, one mask bit per element)"""
    from . import ext
    C = ext()
    OH, OW = OH or H, OW or W
    if out is None:
        out = torch.empty(N, OH, OW, Cb, dtype=torch.float32, device=ap.device)
    # few output tiles (small per-GPU batch): the K loop is split over CTAs, partial tiles summed by a second kernel
    ks = C.conv_fprop_ksplits(N, H, W, Ca, Cb, len(taps), _sm(ap.device)) if KSPLIT else 1
    ws = None
    if ks > 1:
        ws = torch.empty(ks, C.conv_fprop_mtiles(N, H, W) * 128, Cb, dtype=torch.float32, device=ap.device)
    with torch.cuda.device(ap.device):
        C.conv_fprop(ap.data_ptr(), wp.data_ptr(), out.data_ptr(), N, H, W, Ca, Cb, taps, nsrc, wtaps, OH, OW, os_,
                     op, oq, _sm(ap.device), _stream(ap.device), 0 if ws is None else ws.data_ptr(), ks,
                     0 if addend is None else addend.data_ptr(), 0 if addmask is None else addmask.data_ptr())
    return out


def wgrad(xp, gp, N, H, W, Ca, Cb, taps, nsrc=1):
    """dW[co, t, ci] = sum over the pixel grid of X_tap[., ci] * dY[., co]  -> fp32 [Cb, len(taps), Ca]"""
    from . import ext
    C = ext()
    splits = C.conv_wgrad_splits(N, H, W, Ca, Cb, len(taps), _sm(xp.device))
    ws = torch.empty(splits, len(taps) * Ca, Cb, dtype=torch.float32, device=xp.device)
    dw = torch.empty(Cb, len(taps), Ca, dtype=torch.float32, device=xp.device)
    with torch.cuda.device(xp.device):
        C.conv_wgrad(xp.data_ptr(), gp.data_ptr(), ws.data_ptr(), dw.data_ptr(), N, H, W, Ca, Cb, taps, nsrc, splits,
                     _stream(xp.device))
    return dw


# ------------------------------------------------------------------------------------------------ eligibility
def kind_of(x: torch.Tensor, weight: torch.Tensor, stride, padding, dilation, groups):
    """'s1' | 's2' | 'p1' | 'p2' | 'stem' when the tensor-core path applies, else None."""
    if not (enabled() and x.is_cuda and x.dtype == torch.float32 and weight.dtype == torch.float32 and x.dim() == 4):
        return None
    if tuple(dilation) != (1, 1) or groups != 1 or not x.is_contiguous(memory_format=torch.channels_last):
        return None
    from . import ext
    sup = ext().conv_tc_supported
    N, Ci, H, W = x.shape
    Co, k, st, pd = weight.shape[0], tuple(weight.shape[2:]), tuple(stride), tuple(padding)
    if k == (3, 3) and st == (1, 1) and pd == (1, 1):
        if Ci == 3:
            return "stem" if (not x.requires_grad and sup(N, H, W, 64, Co)) else None
        return "s1" if sup(N, H, W, Ci, Co) else None
    if H % 2 or W % 2:
        return None
    if k == (3, 3) and st == (2, 2) and pd == (1, 1):
        return "s2" if sup(N, H // 2, W // 2, Ci, Co) else None
    if k == (1, 1) and st == (2, 2) and pd == (0, 0):
        return "p2" if sup(N, H // 2, W // 2, Ci, Co) else None
    if k == (1, 1) and st == (1, 1) and pd == (0, 0):
        return "p1" if sup(N, H, W, Ci, Co) else None
    return None


def eligible(x, weight, stride, padding, dilation, groups) -> bool:
    return kind_of(x, weight, stride, padding, dilation, groups) is not None


# A down-sampling block feeds the SAME tensor to its 3x3/stride-2 conv and to its 1x1/stride-2 down-sampler: split it
# once.  Only a WEAK reference to the activation is kept: a strong one would keep its autograd graph -- and the
# AccumulateGrad nodes of every earlier layer, bound to the stream of the step that built them -- alive into the
# next step (which breaks CUDA-graph capture); a dead weakref can never match a recycled id().
_PARITY_CACHE = {"ref": None, "ver": -1, "planes": None}


def _parity_planes(x: torch.Tensor) -> torch.Tensor:
    import weakref
    c = _PARITY_CACHE
    if c["ref"] is not None and c["ref"]() is x and c["ver"] == x._version:
        return c["planes"]
    planes = split3_parity(x.permute(0, 2, 3, 1))
    c["ref"], c["ver"], c["planes"] = weakref.ref(x), x._version, planes
    return planes


def conv_forward(x, weight, kind, need_dx):
    """The forward launches of one convolution -> (y [N,OH,OW,Co] fp32, input planes, transposed weight planes or None),
    the planes being what the backward needs."""
    N, Ci, H, W = x.shape
    Co = weight.shape[0]
    w_ohwi = weight.permute(0, 2, 3, 1).contiguous()                   # no copy when the weight is channels_last
    if kind == "stem":
        xp = split3_stem(x.permute(0, 2, 3, 1))
        w64 = F.pad(w_ohwi.reshape(Co, 27), (0, 37)).reshape(Co, 1, 64)
        wp, wtp = wprep(w64, False)
        y = fprop(xp, wp, N, H, W, 64, Co, TAPS_1X1, 1, 1)
    elif kind == "s1":
        xp = planes_get(x)
        if xp is None:
            xp = split3(x)
        wp, wtp = wprep(w_ohwi.reshape(Co, 9, Ci), need_dx)
        y = fprop(xp, wp, N, H, W, Ci, Co, TAPS_S1, 1, 9)
    elif kind == "p1":
        xp = planes_get(x)
        if xp is None:
            xp = split3(x)
        wp, wtp = wprep(w_ohwi.reshape(Co, 1, Ci), need_dx)
        y = fprop(xp, wp, N, H, W, Ci, Co, TAPS_1X1, 1, 1)
    else:                                                               # s2 / p2: parity images of the input
        xp = _parity_planes(x)
        T = 9 if kind == "s2" else 1
        wp, wtp = wprep(w_ohwi.reshape(Co, T, Ci), need_dx)
        y = fprop(xp, wp, N, H // 2, W // 2, Ci, Co, TAPS_S2 if kind == "s2" else TAPS_1X1, 4, T)
    return y, xp, wtp


def conv_backward(xp, wtp, gp, geom, kind, need_dx, need_dw, dev, addend=None, addmask=None, weight=None):
    """Weight gradient (side stream) and data gradient of one convolution from the planes of dY -> (dx, dw).
    addend / addmask (s1 / p1 only): the data gradient becomes dgrad + (mask bit ? addend : 0), in its epilogue.
    weight: the convolution's weight, which decides whether the wait for dw can be deferred (_fork_wgrad.join)."""
    N, Ci, H, W, Co = geom
    dx = dw = None
    if kind == "stem":
        if need_dw:
            d = wgrad(xp, gp, N, H, W, 64, Co, TAPS_1X1, 1)                           # [Co, 1, 64]
            dw = d[:, 0, :27].reshape(Co, 3, 3, 3).permute(0, 3, 1, 2)
    elif kind in ("s1", "p1"):
        taps, dtaps, T = (TAPS_S1, TAPS_S1_DGRAD, 9) if kind == "s1" else (TAPS_1X1, TAPS_1X1, 1)
        fork = _fork_wgrad(dev, PAR_BWD and need_dx and need_dw)
        if need_dw:
            k = 3 if kind == "s1" else 1
            with fork:
                dwr = wgrad(xp, gp, N, H, W, Ci, Co, taps, 1)
            dw = dwr.reshape(Co, k, k, Ci).permute(0, 3, 1, 2)
        if need_dx:
            skip = {} if addend is None else {"addend": addend, "addmask": addmask}
            dx = fprop(gp, wtp, N, H, W, Co, Ci, dtaps, 1, T, **skip).permute(0, 3, 1, 2)
        if need_dw:
            fork.join(dw, weight, xp, gp)
    else:
        assert addend is None, "the skip-connection gradient is folded into stride-1 data gradients only"
        Ho, Wo = H // 2, W // 2
        fork = _fork_wgrad(dev, PAR_BWD and need_dx and need_dw)
        if need_dw:
            k = 3 if kind == "s2" else 1
            with fork:
                dwr = wgrad(xp, gp, N, Ho, Wo, Ci, Co, TAPS_S2 if kind == "s2" else TAPS_1X1, 4)
            dw = dwr.reshape(Co, k, k, Ci).permute(0, 3, 1, 2)
        if need_dx:
            if kind == "s2":
                dxn = torch.empty(N, H, W, Ci, dtype=torch.float32, device=dev)
                for (p, q), taps in TAPS_S2_DGRAD.items():
                    fprop(gp, wtp, N, Ho, Wo, Co, Ci, taps, 1, 9, out=dxn, OH=H, OW=W, os_=2, op=p, oq=q)
            else:                                       # 1x1 stride 2: only the even/even pixels receive a gradient
                dxn = torch.zeros(N, H, W, Ci, dtype=torch.float32, device=dev)
                fprop(gp, wtp, N, Ho, Wo, Co, Ci, TAPS_1X1, 1, 1, out=dxn, OH=H, OW=W, os_=2, op=0, oq=0)
            dx = dxn.permute(0, 3, 1, 2)
        if need_dw:
            fork.join(dw, weight, xp, gp)
    return dx, dw


class _ConvTcFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, kind):
        N, Ci, H, W = x.shape
        ctx.kind, ctx.geom, ctx.weight = kind, (N, Ci, H, W, weight.shape[0]), weakref.ref(weight)
        y, xp, wtp = conv_forward(x, weight, kind, ctx.needs_input_grad[0])
        ctx.save_for_backward(xp, wtp)
        return y.permute(0, 3, 1, 2)                                    # logical NCHW, channels_last memory

    @staticmethod
    def backward(ctx, dy):
        xp, wtp = ctx.saved_tensors
        if dy.dtype != torch.float32 or not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.to(torch.float32).contiguous(memory_format=torch.channels_last)
        gp = planes_get(dy)                                             # emitted by the BN backward that produced dy
        if gp is None:
            gp = split3(dy)
        dx, dw = conv_backward(xp, wtp, gp, ctx.geom, ctx.kind, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                               dy.device, weight=ctx.weight())
        return dx, dw, None


def conv_tc(x: torch.Tensor, weight: torch.Tensor, kind: str) -> torch.Tensor:
    return _ConvTcFn.apply(x, weight, kind)


def conv3x3_tc(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 (kept as the simplest entry point for tests and benchmarks)."""
    return _ConvTcFn.apply(x, weight, "s1")


def conv2d(x: torch.Tensor, weight: torch.Tensor, bias, stride, padding, dilation, groups) -> torch.Tensor:
    """F.conv2d with the tensor-core fp32 path for eligible shapes."""
    if bias is None:
        kind = kind_of(x, weight, stride, padding, dilation, groups)
        if kind is not None:
            return mark_tc_output(_ConvTcFn.apply(x, weight, kind))
    return F.conv2d(x, weight, bias, stride, padding, dilation, groups)


# compatibility helpers for benchmarks/conv_tc_bench.py
def fprop_planes(ap, wp, N, H, W, Ca, Cb):
    return fprop(ap, wp, N, H, W, Ca, Cb, TAPS_S1, 1, 9)


def wgrad_planes(xp, gp, N, H, W, Ca, Cb):
    return wgrad(xp, gp, N, H, W, Ca, Cb, TAPS_S1, 1).reshape(Cb, 3, 3, Ca)
