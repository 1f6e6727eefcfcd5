"""Layer helpers built on the C-ABI kernels: packed convolutions, transposed convolutions as
stride-phase sub-convolutions, linear layers.  Precision follows the activation dtype:
bf16 activations -> wgmma tensor-core kernel, fp32 activations -> fp32 CUDA-core kernel (parity mode).
"""
import torch

from . import ops
from .ops import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_SIGMOID, PackedConv  # noqa: F401


def empty_nhwc(n, h, w, c, dtype, device, c_align=None):
    """NHWC buffer whose pixel stride is padded to 32 bytes: TMA needs 16-byte strides, and 32-byte pixel starts keep the
    epilogue's 256-bit stores and full-sector writes when a layer writes a channel slice of a concat buffer
    (a 176-byte stride for FlowNetFusion's 82-channel concat made conv0 2x slower than the same layer at stride 192)."""
    if c_align is None:
        c_align = 16 if dtype == torch.bfloat16 else 8
    cs = (c + c_align - 1) // c_align * c_align
    buf = torch.empty(n, h, w, cs, dtype=dtype, device=device)
    return buf[..., :c] if cs != c else buf


class Conv:
    """nn.Conv2d (+ folded frozen-BN scale/bias, + activation) on NHWC buffers."""

    def __init__(self, weight, bias=None, stride=1, pad=0, act=ACT_NONE, slope=0.1, scale=None):
        self.pk = PackedConv(weight, bias, scale)
        self.stride, self.pad, self.act, self.slope = stride, pad, act, slope
        self.cout, self.cin = self.pk.cout, self.pk.cin
        self.k = self.pk.kh
        # 3x3 / stride 1 / pad 1 layers with <= 3 output channels (FlowNet2 predict_flow*): in the tc32 precision they run as a
        # 1x1 tensor-core convolution with the taps on the output-channel axis + a 9-tap gather (vps_tap_gather3x3): 9x fewer
        # K steps than the 3x3 implicit GEMM, whose cost does not depend on N
        self.pk_tap = None
        if self.pk.kh == 3 and self.pk.kw == 3 and stride == 1 and pad == 1 and self.cout <= 3:
            w = weight if scale is None else weight * scale.view(-1, 1, 1, 1)
            self.pk_tap = PackedConv(w.permute(2, 3, 0, 1).reshape(9 * self.cout, self.cin, 1, 1).contiguous(), None)

    def out_hw(self, h, w):
        return ((h + 2 * self.pad - self.pk.kh) // self.stride + 1,
                (w + 2 * self.pad - self.pk.kw) // self.stride + 1)

    def tc_ok(self, x):
        # tensor-core path: bf16 activations (or fp32 in the tc32 parity precision) with a 16-byte aligned base and
        # pixel stride (TMA requirement)
        if x.dtype == torch.float32:
            return ops.f32_tc_ok(x)
        return x.dtype == torch.bfloat16 and ops.vt(x).cs % 8 == 0 and x.data_ptr() % 16 == 0

    def __call__(self, x, y=None, act=None, res=None, res_after_act=False, out_scale=1.0, out_dtype=None):
        n, h, w, _ = x.shape
        oh, ow = self.out_hw(h, w)
        if y is None:
            y = empty_nhwc(n, oh, ow, self.cout, out_dtype or x.dtype, x.device)
        act = self.act if act is None else act
        if (x.dtype == torch.bfloat16 or ops.F32_TC[0]) and not self.tc_ok(x):
            # mis-aligned channel slice (e.g. frame 2 of the 6-channel FlowNet input): re-base it once
            xa = empty_nhwc(n, h, w, x.shape[3], x.dtype, x.device)
            ops.copy_scale(x, xa)
            x = xa
        if (self.pk_tap is not None and res is None and x.dtype == torch.float32 and y.dtype == torch.float32
                and ops.F32_TC[0] and self.tc_ok(x)):
            z = empty_nhwc(n, h, w, 9 * self.cout, torch.float32, x.device)
            ops.conv2d(x, self.pk_tap, z, use_tc=True)
            ops.tap_gather3x3(z, y, self.pk.bias, act=act, slope=self.slope, out_scale=out_scale)
            return y
        ops.conv2d(x, self.pk, y, stride=self.stride, pad=self.pad, act=act,
                   slope=self.slope, res=res, res_after_act=res_after_act, out_scale=out_scale,
                   use_tc=self.tc_ok(x))
        return y


class StemConv7x7s2:
    """nn.Conv2d(cin, cout, 7, stride=2, padding=3) for thin inputs (ResNet / FlowNetC / FlowNetS conv1).

    bf16: space-to-depth(2) turns it into a 4x4 stride-1 convolution over 4*cin channels, which the tensor-core
    kernel runs with unit-stride TMA rows (a stride-2 box over 3..12 channels would be a slow element gather):
        in row 2*oy - 3 + r,  r' = r + 1  ->  block row I = oy - 2 + r'//2, parity dy = r' % 2
        W'[co, (dy*2+dx)*cin + c, R, S] = W[co, c, 2R+dy-1, 2S+dx-1]   (0 where an index is -1), padding 2.
    fp32 (parity mode): the plain 7x7 stride-2 CUDA-core convolution."""

    def __init__(self, weight, bias=None, act=ACT_NONE, slope=0.1, scale=None):
        self.plain = Conv(weight, bias, stride=2, pad=3, act=act, slope=slope, scale=scale)
        w = weight if scale is None else weight * scale.view(-1, 1, 1, 1)
        co, ci, _, _ = w.shape
        wp = torch.zeros(co, ci, 8, 8, dtype=torch.float32, device=w.device)
        wp[:, :, 1:, 1:] = w                                   # index r' = r + 1
        w2 = wp.view(co, ci, 4, 2, 4, 2).permute(0, 3, 5, 1, 2, 4).reshape(co, 4 * ci, 4, 4).contiguous()
        self.s2d = Conv(w2, bias, stride=1, pad=2, act=act, slope=slope)
        self.cin, self.cout, self.act = ci, co, act

    def __call__(self, x, y=None, act=None, out_dtype=None):
        if x.dtype != torch.bfloat16 and not ops.F32_TC[0]:
            return self.plain(x, y, act=act, out_dtype=out_dtype)
        n, h, w, c = x.shape
        xs = empty_nhwc(n, (h + 1) // 2, (w + 1) // 2, 4 * c, x.dtype, x.device)
        ops.space_to_depth2(x, xs)
        oh, ow = (h + 6 - 7) // 2 + 1, (w + 6 - 7) // 2 + 1
        if y is None:
            y = empty_nhwc(n, oh, ow, self.cout, out_dtype or x.dtype, x.device)
        # the 4x4/pad-2 conv yields (h/2 + 1) rows; the stride-2 conv defines only the first oh x ow of them
        if ops.PROFILE is not None:
            ops._NOTE["flops_alg"] = 2 * n * oh * ow * self.cout * self.cin * 49
        ops.conv2d(xs, self.s2d.pk, y, stride=1, pad=2, act=self.act if act is None else act, slope=self.s2d.slope,
                   oh=oh, ow=ow, use_tc=True)
        return y


class _PhaseDeconv:
    """ConvTranspose2d(stride 2) as 4 stride-phase convolutions that write interleaved output pixels."""

    def __init__(self, weight_iohw, bias, k):
        # weight_iohw: [cin, cout, k, k] fp32 on device
        self.cin, self.cout = weight_iohw.shape[:2]
        self.k = k
        self._shared32 = None
        self.phases = []
        w_oihw = weight_iohw.permute(1, 0, 2, 3)
        for py in range(2):
            for px in range(2):
                if k == 4:     # padding 1: out[2q+p] taps -> see DESIGN.md "transposed convolutions"
                    ky = [3, 1] if py == 0 else [2, 0]
                    kx = [3, 1] if px == 0 else [2, 0]
                    sub = w_oihw[:, :, ky][:, :, :, kx].contiguous()
                    pad = (1 - py, 1 - px)
                else:          # k == 2, padding 0: out[2q+p] = x[q] * w[p]
                    sub = w_oihw[:, :, py:py + 1, px:px + 1].contiguous()
                    pad = (0, 0)
                self.phases.append((py, px, pad, PackedConv(sub, bias)))

    def __call__(self, x, y, act=ACT_NONE, slope=0.1, out_scale=1.0):
        n, h, w, _ = x.shape
        use_tc = (x.dtype == torch.bfloat16 and self.cin >= 16 and ops.vt(x).cs % 8 == 0
                  and x.data_ptr() % 16 == 0) or (self.cin >= 16 and ops.f32_tc_ok(x))
        if use_tc:      # all four stride phases in one persistent launch
            if x.dtype == torch.float32 and self._shared32 is None:
                self._shared32 = ops.pack_tc32([ph[3] for ph in self.phases])
            ops.conv2d_tc_multi(x, [ph[3] for ph in self.phases], y, [ph[2] for ph in self.phases],
                                [(2, ph[0], 2, ph[1]) for ph in self.phases], act=act, slope=slope,
                                out_scale=out_scale, oh=h, ow=w, shared32=self._shared32)
            return y
        for py, px, pad, pk in self.phases:
            ops.conv2d(x, pk, y, stride=1, pad_hw=pad, act=act, slope=slope, oh=h, ow=w,
                       omap=(2, py, 2, px), out_scale=out_scale, use_tc=False)
        return y


def deconv4x4_s2(weight_iohw, bias):
    """nn.ConvTranspose2d(cin, cout, 4, 2, 1) -- FlowNet2 `deconv` / `upsampled_flow*` (submodules.py:33-37)."""
    return _PhaseDeconv(weight_iohw, bias, 4)


def deconv2x2_s2(weight_iohw, bias):
    """nn.ConvTranspose2d(cin, cout, 2, stride=2) -- FCNMaskHead.upsample (fcn_mask_head.py:66-71)."""
    return _PhaseDeconv(weight_iohw, bias, 2)


class Linear:
    """nn.Linear over rows: x viewed as NHWC [1,1,M,K]."""

    def __init__(self, weight, bias=None, act=ACT_NONE):
        self.pk = PackedConv(weight.view(weight.shape[0], weight.shape[1], 1, 1), bias)
        self.act = act
        self.cout = weight.shape[0]

    def __call__(self, x2d, y2d=None, out_dtype=None):
        m, k = x2d.shape
        if y2d is None:
            y2d = torch.empty(m, (self.cout + 7) // 8 * 8, dtype=out_dtype or x2d.dtype, device=x2d.device)[:, :self.cout]
        x4 = x2d.unsqueeze(0).unsqueeze(0)
        y4 = y2d.unsqueeze(0).unsqueeze(0)
        use_tc = (x2d.dtype == torch.bfloat16 and x2d.stride(0) % 8 == 0 and x2d.data_ptr() % 16 == 0) or ops.f32_tc_ok(x4)
        ops.conv2d(x4, self.pk, y4, act=self.act, use_tc=use_tc)
        return y2d
