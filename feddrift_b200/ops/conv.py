"""``TcConv2d`` — nn.Conv2d-compatible layer whose CUDA path is the hand-written IMPLICIT-GEMM convolution on wgmma:
forward, data gradient and weight gradient, NHWC activations end to end.  Two kernel families, picked per direction by shape:

* **TMA-im2col path** (``csrc/gemm_tc.cu`` conv modes; Cin % 64 == 0, square filter, symmetric padding — every body layer of
  the ResNets): activations are cast once to bf16 NHWC and the persistent GEMM mainloop's producer thread fetches the operand
  tiles with ``cp.async.bulk.tensor.4d…im2col`` — the TMA unit walks the output pixels (conv stride = traversal stride), applies
  the filter-tap offset and zero-fills the halo; no gather code runs on the SMs.  Forward = A[pixel,(tap,c)]·Wᵀ with the
  bias(+ReLU) epilogue; stride-1 data gradient = the same kernel on dY with the tap-flipped transposed weight pack; weight
  gradient = a GEMM over the pixels whose B operand is an MN-major im2col box and whose A operand is dY as it lies in memory,
  split over pixel ranges with ``cp.reduce.async.bulk`` adds.
* **software-gather path** (``csrc/conv_igemm.cu``; Cin, Cout % 32 == 0): producer warps gather each pixel's (tap, channel)
  slice from the fp32 NHWC tensor into no-swizzle operand tiles; used for 32-channel layers and strided data gradients.

fp32 activations / master weights, bf16 tensor-core operands, fp32 accumulation; results are NCHW *views* with
channels_last strides, so a chain of convolutions never transposes.  Shapes neither family covers (groups / dilation ≠ 1,
1- or 3-channel stems) and CPU tensors use ``F.conv2d``.  State-dict keys and the init law equal ``nn.Conv2d``'s.
Reference: cuDNN fp32 ``nn.Conv2d`` (``fedml_api/model/cv/cnn.py:110-117``).
"""
from __future__ import annotations

import math
import os

import torch
import torch.nn.functional as F
from torch import nn

from . import _ext
from ..models.utils import ohwi_stored as _ohwi

TC_CONV_CALLS = 0
IGEMM_CALLS = {"fwd": 0, "dgrad": 0, "wgrad": 0, "tma_fwd": 0, "tma_dgrad": 0, "tma_wgrad": 0}


def _pair(v):
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def _nhwc(t: torch.Tensor) -> torch.Tensor:
    """Contiguous NHWC view of an NCHW-logical tensor (free when it already is channels_last)."""
    return t.float().contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)


def igemm_eligible(cin: int, cout: int, stride, dilation, groups: int) -> bool:
    # forward needs Cin % 16 / Cout % 32; the data gradient swaps the roles → both multiples of 32
    return groups == 1 and tuple(dilation) == (1, 1) and stride[0] == stride[1] and cin % 32 == 0 and cout % 32 == 0


def tma_eligible(cin: int, stride, padding, ksize) -> bool:
    """The GEMM-mainloop path with the TMA-im2col producer: 64-channel K chunks, square filter, symmetric padding."""
    return (cin % 64 == 0 and ksize[0] == ksize[1] and padding[0] == padding[1] and stride[0] == stride[1] and 1 <= stride[0] <= 8
            and padding[0] < 128)


def _nhwc_bf16(ext, t: torch.Tensor, gate=None) -> torch.Tensor:
    """bf16 NHWC copy of an NCHW-logical fp32 tensor: our cast kernel when the memory already is channels_last (optionally
    fused with the ReLU-backward gate), one fused layout+dtype copy otherwise."""
    if t.dtype == torch.float32 and t.is_contiguous(memory_format=torch.channels_last):
        return ext.conv_cast_bf16(t.permute(0, 2, 3, 1), gate)
    tb = t.to(dtype=torch.bfloat16, memory_format=torch.channels_last).permute(0, 2, 3, 1)
    return tb if gate is None else tb * (gate > 0)


def _weight_ohwi(weight: torch.Tensor) -> torch.Tensor:
    """fp32 [Cout, kh, kw, Cin] contiguous: a free view when the parameter is stored channels_last (the flat-row layout of
    ``models.utils.flat_view`` and the layout ``TcConv2d`` allocates), one transposing copy otherwise."""
    w = weight.detach()
    if w.dtype != torch.float32:
        w = w.float()
    return w.permute(0, 2, 3, 1).contiguous()       # no-op for channels_last storage


def _dilate(gb: torch.Tensor, stride: int, H: int, W: int, k: int, pad: int) -> torch.Tensor:
    """Strided layers: dY (bf16 NHWC) with ``stride-1`` zeros between the pixels, sized so that the stride-1 data-gradient
    convolution returns exactly ``[H, W]`` — the strided data gradient then runs on the same TMA-im2col kernel (3/4 of its
    multiply-adds hit zeros, which is still several times faster than the software gather it replaces)."""
    if stride == 1:
        return gb
    N, P, Q, C = gb.shape
    out = gb.new_zeros(N, H - k + 1 + 2 * pad, W - k + 1 + 2 * pad, C)
    out[:, 0:(P - 1) * stride + 1:stride, 0:(Q - 1) * stride + 1:stride] = gb
    return out


class _ConvIgemmFn(torch.autograd.Function):
    """Implicit-GEMM convolution.  Per direction the kernel is picked by shape: the GEMM mainloop with a TMA-im2col producer
    (``gemm_tc.cu`` conv modes; bf16 NHWC operands, Cin % 64 == 0 — every body layer of the ResNets) or the software-gather
    kernels of ``conv_igemm.cu`` (Cin % 32, strided data gradients).  The weight operand of forward AND data gradient is one
    bf16 cast of the channels_last parameter; the weight gradient is reduce-added into the channels_last ``.grad`` in place."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, relu: bool):
        global TC_CONV_CALLS
        TC_CONV_CALLS += 1
        IGEMM_CALLS["fwd"] += 1
        ext = _ext.load(required=True)
        Co, Ci, kh, kw = weight.shape
        wq = ext.conv_cast_bf16(_weight_ohwi(weight), None)            # bf16 [Cout][kh][kw][Cin]
        bdet = bias.detach() if bias is not None else None
        tma_in = tma_eligible(Ci, stride, padding, (kh, kw))          # forward and weight gradient gather from x
        if tma_in:
            IGEMM_CALLS["tma_fwd"] += 1
            xs = _nhwc_bf16(ext, x)
            y = ext.conv_tma_fwd(xs, wq, bdet, stride[0], padding[0], bool(relu), 1)
        else:
            xs = _nhwc(x)
            y = ext.conv_igemm_fwd(xs, wq, bdet, stride[0], padding[0], padding[1], bool(relu))
        ctx.save_for_backward(xs, wq, y if relu else None)
        ctx.weight_ref = weight if isinstance(weight, torch.nn.Parameter) else None
        ctx.geom = (stride, padding, tuple(weight.shape), tuple(x.shape[2:]))
        ctx.relu, ctx.has_bias, ctx.tma_in = relu, bias is not None, tma_in
        return y.permute(0, 3, 1, 2)                                          # NCHW view, channels_last strides

    @staticmethod
    def backward(ctx, gy):
        ext = _ext.load(required=True)
        xs, wq, y = ctx.saved_tensors
        stride, padding, (Co, Ci, kh, kw), (H, W) = ctx.geom
        tma_dgrad = ctx.needs_input_grad[0] and padding[0] <= kh - 1 and tma_eligible(Co, stride, padding, (kh, kw))
        tma_wgrad = ctx.needs_input_grad[1] and ctx.tma_in
        need_f32 = ((ctx.needs_input_grad[0] and not tma_dgrad) or (ctx.needs_input_grad[1] and not tma_wgrad)
                    or (ctx.has_bias and ctx.needs_input_grad[2]))
        g = gb = None
        if need_f32:
            g = _nhwc(gy)
            if ctx.relu:
                g = g * (y > 0)
        if tma_dgrad or tma_wgrad:
            gb = ext.conv_cast_bf16(g, None) if g is not None else _nhwc_bf16(ext, gy, y if ctx.relu else None)
        gx = gw = gbias = None
        if ctx.needs_input_grad[0]:
            IGEMM_CALLS["dgrad"] += 1
            if tma_dgrad:      # data gradient = stride-1 convolution of (zero-dilated) dY; the forward pack is read MN-major, taps flipped
                IGEMM_CALLS["tma_dgrad"] += 1
                gx = ext.conv_tma_dgrad(_dilate(gb, stride[0], H, W, kh, padding[0]), wq, padding[0], 1).permute(0, 3, 1, 2)
            else:
                gx = ext.conv_igemm_dgrad(g, ext.conv_pack_t(wq), H, W, stride[0], padding[0], padding[1]).permute(0, 3, 1, 2)
        if ctx.needs_input_grad[1]:
            IGEMM_CALLS["wgrad"] += 1
            wp = ctx.weight_ref
            acc = None
            if (wp is not None and wp.grad is not None and wp.grad.is_cuda and wp.grad.dtype == torch.float32 and wp.grad.shape == wp.shape
                    and wp.grad.is_contiguous(memory_format=torch.channels_last)):
                # a preallocated channels_last .grad (the federated executor binds every parameter's .grad to its segment of the
                # flat, zeroed gradient row): the kernel reduce-adds straight into it — no zero-fill, no AccumulateGrad launch
                acc = wp.grad.permute(0, 2, 3, 1)
            buf = acc if acc is not None else torch.zeros(Co, kh, kw, Ci, dtype=torch.float32, device=xs.device)
            if tma_wgrad:
                IGEMM_CALLS["tma_wgrad"] += 1
                ext.conv_tma_wgrad(xs, gb, buf, kh, stride[0], padding[0], 1)
            else:
                ext.conv_igemm_wgrad(xs, g, kh, kw, stride[0], padding[0], padding[1], buf, True)
            gw = None if acc is not None else buf.permute(0, 3, 1, 2)          # logical OIHW view of the channels_last buffer
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gbias = g.sum((0, 1, 2))
        return gx, gw, gbias, None, None, None


def stacked_eligible(layer, x: torch.Tensor) -> bool:
    """Grouped (one group per stacked pair) implicit-GEMM path of ``sim/stacked.py::StackedConv2d``: all three directions on the
    TMA-im2col GEMM kernels, which needs 64-channel chunks on both sides."""
    return (x.is_cuda and x.dim() == 4 and layer.groups == 1 and layer.dilation == (1, 1) and layer.in_channels % 64 == 0
            and layer.out_channels % 64 == 0 and layer.padding[0] <= layer.kernel_size[0] - 1
            and tma_eligible(layer.in_channels, layer.stride, layer.padding, layer.kernel_size)
            and os.environ.get("FDB_NO_TC_CONV") != "1" and _ext.available() and hasattr(_ext.load(), "conv_cast_rows_bf16"))


def _rows2d(w: torch.Tensor):
    """[n, Co, Ci, kh, kw] strided view of the staged rows (each pair's weight channels_last) → the [n, Co·kh·kw·Ci] rows view."""
    n = w.shape[0]
    v = w.permute(0, 1, 3, 4, 2)
    r = v.reshape(n, -1)
    return r if r.stride(1) == 1 and r.data_ptr() == w.data_ptr() else None


class _StackedConvFn(torch.autograd.Function):
    """Grouped implicit-GEMM convolution over ``n`` stacked (client, model) pairs: ``x`` is ``[B, n·Ci, H, W]``, ``weight`` the
    strided view ``[n, Co, Ci, kh, kw]`` of the staged parameter rows.  One cast kernel turns all pairs' weights into the bf16
    operand, forward / data gradient are ONE launch each for all pairs, and the weight gradients are reduce-added straight into
    the pairs' gradient rows through a 3-D tensor map (``weight.grad`` is the matching strided view)."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, relu: bool, n: int):
        global TC_CONV_CALLS
        TC_CONV_CALLS += 1
        IGEMM_CALLS["stacked_fwd"] = IGEMM_CALLS.get("stacked_fwd", 0) + 1
        ext = _ext.load(required=True)
        _, Co, Ci, kh, kw = weight.shape
        w2 = _rows2d(weight.detach())
        if w2 is None:
            w2 = weight.detach().permute(0, 1, 3, 4, 2).reshape(n, -1).contiguous()
        wq = ext.conv_cast_rows_bf16(w2).view(n * Co, kh, kw, Ci)
        xb = _nhwc_bf16(ext, x)
        b = bias.detach().reshape(-1) if bias is not None else None
        y = ext.conv_tma_fwd(xb, wq, b, stride[0], padding[0], bool(relu), n)
        ctx.save_for_backward(xb, wq, y if relu else None)
        ctx.weight_ref = weight if isinstance(weight, torch.nn.Parameter) else None
        ctx.geom = (stride, padding, (n, Co, Ci, kh, kw), tuple(x.shape[2:]))
        ctx.relu, ctx.has_bias = relu, bias is not None
        return y.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, gy):
        ext = _ext.load(required=True)
        xb, wq, y = ctx.saved_tensors
        stride, padding, (n, Co, Ci, kh, kw), (H, W) = ctx.geom
        g = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            g = _nhwc(gy)
            if ctx.relu:
                g = g * (y > 0)
        gb = ext.conv_cast_bf16(g, None) if g is not None else _nhwc_bf16(ext, gy, y if ctx.relu else None)
        gx = gw = gbias = None
        if ctx.needs_input_grad[0]:
            gx = ext.conv_tma_dgrad(_dilate(gb, stride[0], H, W, kh, padding[0]), wq, padding[0], n).permute(0, 3, 1, 2)
        if ctx.needs_input_grad[1]:
            wp = ctx.weight_ref
            acc = _rows2d(wp.grad) if (wp is not None and wp.grad is not None and wp.grad.shape == wp.shape and wp.grad.dtype == torch.float32) else None
            buf = acc if acc is not None else torch.zeros(n, Co * kh * kw * Ci, dtype=torch.float32, device=xb.device)
            if n == 1:
                ext.conv_tma_wgrad(xb, gb, buf.view(Co, kh, kw, Ci), kh, stride[0], padding[0], 1)
            else:
                ext.conv_tma_wgrad(xb, gb, buf, kh, stride[0], padding[0], n)
            gw = None if acc is not None else buf.view(n, Co, kh, kw, Ci).permute(0, 1, 4, 2, 3)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gbias = g.sum((0, 1, 2)).view(n, Co)
        return gx, gw, gbias, None, None, None, None


class TcConv2d(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, kernel_size, stride=1, padding=0, dilation=1, groups: int = 1,
                 bias: bool = True, activation: str = "none"):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding = _pair(kernel_size), _pair(stride), _pair(padding)
        self.dilation, self.groups, self.activation = _pair(dilation), groups, activation
        # channels_last storage ([Cout][kh][kw][Cin]) = the K-major operand layout of the implicit-GEMM kernels = the layout of
        # the flat parameter rows for these shapes (models.utils.ohwi_stored)
        w = torch.empty(out_channels, in_channels // groups, *self.kernel_size)
        self.weight = nn.Parameter(w.contiguous(memory_format=torch.channels_last) if _ohwi(w.shape) else w)
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self) -> None:  # identical init law to nn.Conv2d
        w = torch.empty(self.weight.shape)                    # drawn in logical order: same values as nn.Conv2d for a given seed
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        with torch.no_grad():
            self.weight.copy_(w)
        if self.bias is not None:
            fan_in = self.weight.shape[1] * self.kernel_size[0] * self.kernel_size[1]
            bound = 1 / math.sqrt(fan_in) if fan_in > 0 else 0
            nn.init.uniform_(self.bias, -bound, bound)

    def _use_igemm(self, x: torch.Tensor) -> bool:
        return (x.is_cuda and x.dim() == 4 and _ext.available() and os.environ.get("FDB_NO_TC_CONV") != "1"
                and hasattr(_ext.load(), "conv_igemm_fwd")
                and igemm_eligible(self.in_channels, self.out_channels, self.stride, self.dilation, self.groups))

    def forward(self, x):
        relu = self.activation == "relu"
        if self._use_igemm(x):
            return _ConvIgemmFn.apply(x, self.weight, self.bias, self.stride, self.padding, relu)
        w = self.weight
        if not x.is_cuda:       # CPU: canonical (contiguous NCHW) formats only — see models.utils.unflatten_to_state_dict
            x, w = x.contiguous(), w.contiguous()
        y = F.conv2d(x, w, self.bias, self.stride, self.padding, self.dilation, self.groups)
        return F.relu(y) if relu else y

    def extra_repr(self) -> str:
        return (f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, "
                f"padding={self.padding}, activation={self.activation}")


def convert_convs_(module: nn.Module) -> nn.Module:
    """Replace every ``nn.Conv2d`` of ``module`` whose shape the tensor-core kernels take — or whose weight the flat rows store
    channels_last (``models.utils.ohwi_stored``; ``TcConv2d`` is the layer that consumes that layout safely on CPU too) — in place
    by a :class:`TcConv2d` with the same parameter values; state-dict keys, shapes and values are unchanged.  Used for the torchvision / model-zoo networks so that their 3×3 and
    1×1 body convolutions run on the implicit-GEMM wgmma kernels (stems with 1 or 3 input channels stay library convs)."""
    for name, child in list(module.named_children()):
        if isinstance(child, nn.Conv2d) and type(child).forward is nn.Conv2d.forward and child.padding_mode == "zeros" \
                and not isinstance(child.padding, str) and \
                (igemm_eligible(child.in_channels, child.out_channels, _pair(child.stride), _pair(child.dilation), child.groups)
                 or _ohwi(child.weight.shape)):
            tc = TcConv2d(child.in_channels, child.out_channels, child.kernel_size, child.stride, child.padding, child.dilation,
                          child.groups, bias=child.bias is not None)
            wd = child.weight.detach()
            tc.weight = nn.Parameter(wd.contiguous(memory_format=torch.channels_last) if _ohwi(wd.shape) else wd,
                                     requires_grad=child.weight.requires_grad)
            tc.bias = child.bias
            setattr(module, name, tc)
        else:
            convert_convs_(child)
    return module
