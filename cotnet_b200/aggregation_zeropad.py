"""Drop-in for the reference's ``cupy_layers/aggregation_zeropad.py`` operator API.

Same names, signatures, shapes and error behaviour as the reference
(/root/reference/cupy_layers/aggregation_zeropad.py):
    AggregationZeropad.apply(input, weight, kernel_size, stride, padding, dilation)   :112-186
    aggregation_zeropad(input, weight, kernel_size=3, stride=1, padding=0, dilation=1)  :188-197
    LocalConvolution(in_channels, out_channels, kernel_size, stride, padding, dilation, pad_mode)  :199-236
but the kernels are the sm_90a ones in libcotb200.so reached through the C ABI (include/cotb200.h);
dimensions are runtime arguments, so there is no per-shape NVRTC compile.

Extensions over the reference (which is fp32/fp64 + NCHW-contiguous only, utils.py:8-12):
  * bfloat16 / float16 tensors (fp32 accumulation);
  * channels_last inputs run natively (NHWC kernels), returning a channels_last output -- the reference
    silently mis-indexes such tensors (``clone()`` keeps channels_last strides, :125-128).
"""
import torch
from torch import Tensor
from torch.autograd import Function
from torch.nn.modules.utils import _pair

from . import _lib


def _out_hw(H, W, k, s, p, d):
    # aggregation_zeropad.py:119-120
    Ho = int((H + 2 * p[0] - (d[0] * (k[0] - 1) + 1)) / s[0] + 1)
    Wo = int((W + 2 * p[1] - (d[1] * (k[1] - 1) + 1)) / s[1] + 1)
    return Ho, Wo


def _is_nhwc(x: Tensor, w: Tensor) -> bool:
    """True when x is channels_last-dense and w is the matching NHWC view ([N,Ho,Wo,heads,wc,K2] in memory)."""
    if x.is_contiguous():
        return False
    return x.is_contiguous(memory_format=torch.channels_last) and w.permute(0, 4, 5, 1, 2, 3).is_contiguous()


def _desc(x, w, k, s, p, d, Ho, Wo, layout, fold=1):
    dsc = _lib.AggDesc()
    dsc.n, dsc.c, dsc.h, dsc.w = x.shape
    dsc.heads, dsc.wc = w.shape[1], w.shape[2]
    dsc.kh, dsc.kw = k
    dsc.sh, dsc.sw = s
    dsc.ph, dsc.pw = p
    dsc.dh, dsc.dw = d
    dsc.ho, dsc.wo = Ho, Wo
    dsc.dtype = _lib.dtype_code(x)
    dsc.layout = layout
    dsc.fold = fold
    return dsc


class AggregationZeropad(Function):
    @staticmethod
    def forward(ctx, input, weight, kernel_size, stride, padding, dilation, fold=1):
        # `fold` (extension, default 1 == reference behaviour): CoXt channel fold, see include/cotb200.h
        kernel_size, stride, padding, dilation = _pair(kernel_size), _pair(stride), _pair(padding), _pair(dilation)
        ctx.kernel_size, ctx.stride, ctx.padding, ctx.dilation = kernel_size, stride, padding, dilation
        ctx.fold = fold
        assert input.dim() == 4 and input.is_cuda and weight.is_cuda
        assert weight.dim() == 6 and weight.dtype == input.dtype and weight.device == input.device
        batch_size, input_channels, input_height, input_width = input.size()
        _, weight_heads, weight_channels, weight_kernels, weight_height, weight_width = weight.size()
        assert weight_kernels == kernel_size[0] * kernel_size[1]
        output_height, output_width = _out_hw(input_height, input_width, kernel_size, stride, padding, dilation)
        assert output_height * output_width == weight_height * weight_width
        input, weight = input.detach(), weight.detach()
        nhwc = _is_nhwc(input, weight)
        if nhwc:
            output = torch.empty((batch_size, weight_heads * input_channels, output_height, output_width),
                                 dtype=input.dtype, device=input.device, memory_format=torch.channels_last)
        else:
            input, weight = input.contiguous(), weight.contiguous()
            output = input.new_empty((batch_size, weight_heads * input_channels, output_height, output_width))
        dsc = _desc(input, weight, kernel_size, stride, padding, dilation, output_height, output_width,
                    _lib.NHWC if nhwc else _lib.NCHW, fold)
        if output.numel():
            with torch.cuda.device_of(input):
                rc = _lib.load().cotb200_agg_zeropad_fwd(dsc, input.data_ptr(), weight.data_ptr(), output.data_ptr(),
                                                         _lib.stream_ptr(input))
            _lib.check(rc, "agg_zeropad_fwd")
        ctx.save_for_backward(input, weight)
        ctx.nhwc = nhwc
        ctx.out_hw = (output_height, output_width)
        return output

    @staticmethod
    def backward(ctx, grad_output):
        input, weight = ctx.saved_tensors
        assert grad_output.is_cuda
        nhwc = ctx.nhwc
        if nhwc:
            grad_output = grad_output.contiguous(memory_format=torch.channels_last)
        else:
            grad_output = grad_output.contiguous()
        grad_input = grad_weight = None
        if ctx.needs_input_grad[0]:
            grad_input = torch.empty_like(input)          # preserves NCHW / channels_last
        if ctx.needs_input_grad[1]:
            grad_weight = torch.empty_like(weight)        # preserves the NHWC view strides
        if (grad_input is not None or grad_weight is not None) and grad_output.numel():
            dsc = _desc(input, weight, ctx.kernel_size, ctx.stride, ctx.padding, ctx.dilation, ctx.out_hw[0],
                        ctx.out_hw[1], _lib.NHWC if nhwc else _lib.NCHW, ctx.fold)
            with torch.cuda.device_of(input):
                rc = _lib.load().cotb200_agg_zeropad_bwd(dsc, grad_output.data_ptr(), input.data_ptr(), weight.data_ptr(),
                                                         _lib.ptr(grad_input), _lib.ptr(grad_weight),
                                                         _lib.stream_ptr(input))
            _lib.check(rc, "agg_zeropad_bwd")
        return grad_input, grad_weight, None, None, None, None, None


def aggregation_zeropad(input, weight, kernel_size=3, stride=1, padding=0, dilation=1):
    assert input.shape[0] == weight.shape[0] and (input.shape[1] % weight.shape[2] == 0)
    if input.is_cuda:
        out = AggregationZeropad.apply(input, weight, kernel_size, stride, padding, dilation)
    else:
        # the reference's only "CPU path": bounce through the GPU (aggregation_zeropad.py:192-196)
        if not torch.cuda.is_available():
            raise RuntimeError("cotb200 aggregation_zeropad: CPU tensors are bounced through the GPU like the "
                               "reference does, but no CUDA device is available (there is no CPU implementation)")
        out = AggregationZeropad.apply(input.cuda(), weight.cuda(), kernel_size, stride, padding, dilation)
        torch.cuda.synchronize()
        out = out.cpu()
    return out


class LocalConvolution(torch.nn.Module):
    """Same constructor / attributes as the reference module (aggregation_zeropad.py:199-236);
    ``utils/flops_counter.py:493-509,614`` reads ``kernel_size`` and ``in_channels`` from it."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int, stride: int = 1, padding: int = 0,
                 dilation: int = 1, pad_mode: int = 0):
        super(LocalConvolution, self).__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = kernel_size
        self.stride = stride
        self.padding = padding
        self.dilation = dilation
        self.pad_mode = pad_mode

    def forward(self, input: Tensor, weight: Tensor):
        return aggregation_zeropad(input, weight, kernel_size=self.kernel_size, stride=self.stride,
                                   padding=self.padding, dilation=self.dilation)

    def extra_repr(self):
        return "in_channels=%d, out_channels=%d, kernel_size=%s, stride=%s, padding=%s, dilation=%s" % (
            self.in_channels, self.out_channels, self.kernel_size, self.stride, self.padding, self.dilation)
