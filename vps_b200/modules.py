"""vps_b200 modules registered under the reference's registry names (the host-side mirror of the
reference's plugin interface for the FuseTrack path).

Every class takes the constructor kwargs of its reference namesake (configs/cityscapes/fusetrack.py:2-86),
owns parameters under the reference's state_dict names (so `latest.pth`-style checkpoints load with
strict=True), and runs its forward entirely through libvps_b200.so on NHWC device buffers.  torch.nn is
used only as a parameter container; no torch arithmetic runs on the data path.

`prepare()` packs the parameters into kernel layouts (frozen BN folded into the conv, FC columns
permuted to the NHWC RoI layout, DCN weights tap-major, fused sibling heads); it runs lazily and must be
re-run (`prepare(force=True)`) after loading new weights.
"""
import math

import torch
import torch.nn as nn

from . import ops
from .layers import (ACT_LRELU, ACT_NONE, ACT_RELU, Conv, Linear, StemConv7x7s2, deconv2x2_s2, deconv4x4_s2, empty_nhwc)
from .registry import (BACKBONES, EXTRA_NECKS, HEADS, LOSSES, NECKS, PANOPTIC, ROI_EXTRACTORS, build_loss)


class _Prepared(nn.Module):
    """Parameter holder with lazily packed kernel-side weights."""

    def __init__(self):
        super().__init__()
        self._packed = False

    def prepare(self, force=False):
        if self._packed and not force:
            return self
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("%s: parameters must be on a CUDA device (there is no CPU path)" % type(self).__name__)
        with torch.no_grad():
            self._pack()
        self._packed = True
        return self

    def _pack(self):
        raise NotImplementedError

    def init_weights(self, pretrained=None):
        pass


def _bn_fold(bn):
    scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    return scale, bn.bias - bn.running_mean * scale


def _conv(m, stride=None, pad=None, act=ACT_NONE, bn=None, slope=0.1):
    """nn.Conv2d (+ optional frozen BN) -> packed Conv."""
    scale, bias = (None, m.bias)
    if bn is not None:
        scale, bias = _bn_fold(bn)
        if m.bias is not None:
            bias = bias + m.bias * scale
    return Conv(m.weight.detach(), None if bias is None else bias.detach(), stride=m.stride[0] if stride is None else stride,
                pad=m.padding[0] if pad is None else pad, act=act, slope=slope,
                scale=None if scale is None else scale.detach())


# ============================================================================ losses (built by heads even at test)
@LOSSES.register_module
class CrossEntropyLoss(nn.Module):
    """Constructor-compatible stub of mmdet/models/losses/cross_entropy_loss.py:67-108 (training is a later row)."""

    def __init__(self, use_sigmoid=False, use_mask=False, loss_weight=1.0):
        super().__init__()
        self.use_sigmoid, self.use_mask, self.loss_weight = use_sigmoid, use_mask, loss_weight

    def forward(self, *a, **k):
        raise NotImplementedError("training losses are out of scope of the inference path (SURVEY 8f rank 3)")


@LOSSES.register_module
class SmoothL1Loss(nn.Module):
    def __init__(self, beta=1.0, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.beta, self.reduction, self.loss_weight = beta, reduction, loss_weight

    def forward(self, *a, **k):
        raise NotImplementedError("training losses are out of scope of the inference path (SURVEY 8f rank 3)")


# ============================================================================ backbone
class _Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride, downsample):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        if downsample:
            self.downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False),
                                            nn.BatchNorm2d(planes * 4))
        else:
            self.downsample = None


@BACKBONES.register_module
class ResNet(_Prepared):
    """mmdet/models/backbones/resnet.py:333-526 (depth 50/101/152, pytorch style, eval-mode BN folded)."""
    arch_settings = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}

    def __init__(self, depth, num_stages=4, strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3),
                 style='pytorch', frozen_stages=-1, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True),
                 norm_eval=True, dcn=None, stage_with_dcn=(False, False, False, False), gcb=None,
                 stage_with_gcb=(False, False, False, False), gen_attention=None,
                 stage_with_gen_attention=((), (), (), ()), with_cp=False, zero_init_residual=True):
        super().__init__()
        if depth not in self.arch_settings:
            raise KeyError('invalid depth {} for resnet'.format(depth))
        assert style == 'pytorch' and dcn is None and gcb is None and gen_attention is None, \
            "only the configuration used by fusetrack.py is implemented"
        assert tuple(dilations[:num_stages]) == (1,) * num_stages
        self.out_indices = out_indices
        self.num_stages = num_stages
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        inplanes = 64
        for i, blocks in enumerate(self.arch_settings[depth][:num_stages]):
            planes = 64 * 2 ** i
            layers = [_Bottleneck(inplanes, planes, strides[i], True)]
            inplanes = planes * 4
            layers += [_Bottleneck(inplanes, planes, 1, False) for _ in range(1, blocks)]
            setattr(self, 'layer%d' % (i + 1), nn.Sequential(*layers))

    def _pack(self):
        sc, sh = _bn_fold(self.bn1)
        self.k_stem = StemConv7x7s2(self.conv1.weight.detach(), sh.detach(), act=ACT_RELU, scale=sc.detach())
        self.k_layers = []
        for i in range(self.num_stages):
            blocks = []
            for b in getattr(self, 'layer%d' % (i + 1)):
                blocks.append(dict(
                    c1=_conv(b.conv1, act=ACT_RELU, bn=b.bn1), c2=_conv(b.conv2, act=ACT_RELU, bn=b.bn2),
                    c3=_conv(b.conv3, act=ACT_RELU, bn=b.bn3),
                    ds=None if b.downsample is None else _conv(b.downsample[0], act=ACT_NONE, bn=b.downsample[1])))
            self.k_layers.append(blocks)

    def forward(self, x):
        """x: NHWC [n,H,W,3] -> tuple of NHWC stage outputs."""
        self.prepare()
        x = self.k_stem(x)
        n, h, w, c = x.shape
        y = empty_nhwc(n, (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1, c, x.dtype, x.device)
        ops.pool2d(x, y, 3, 2, 1)
        x = y
        outs = []
        for i, blocks in enumerate(self.k_layers):
            for b in blocks:
                identity = x if b['ds'] is None else b['ds'](x)
                t = b['c2'](b['c1'](x))
                x = b['c3'](t, res=identity)          # relu(bn3(conv3) + identity), resnet.py:236-258
            if i in self.out_indices:
                outs.append(x)
        return tuple(outs)


# ============================================================================ FPN
class _ConvModule(nn.Module):
    """parameter holder matching ConvModule (conv_module.py:44-166): `.conv`."""

    def __init__(self, cin, cout, k, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, padding=padding, bias=True)


@NECKS.register_module
class FPN(_Prepared):
    """mmdet/models/necks/fpn.py:10-139 (no extra convs, no activation)."""

    def __init__(self, in_channels, out_channels, num_outs, start_level=0, end_level=-1, add_extra_convs=False,
                 extra_convs_on_inputs=True, relu_before_extra_convs=False, conv_cfg=None, norm_cfg=None,
                 activation=None):
        super().__init__()
        assert isinstance(in_channels, list) and start_level == 0 and end_level == -1 and not add_extra_convs
        assert activation is None and norm_cfg is None
        self.in_channels, self.out_channels, self.num_outs = in_channels, out_channels, num_outs
        self.lateral_convs = nn.ModuleList([_ConvModule(c, out_channels, 1) for c in in_channels])
        self.fpn_convs = nn.ModuleList([_ConvModule(out_channels, out_channels, 3, 1) for _ in in_channels])

    def _pack(self):
        self.k_lat = [_conv(m.conv) for m in self.lateral_convs]
        self.k_out = [_conv(m.conv) for m in self.fpn_convs]

    def forward(self, inputs):
        self.prepare()
        lat = [k(inputs[i]) for i, k in enumerate(self.k_lat)]
        for i in range(len(lat) - 1, 0, -1):                       # fpn.py:110-113 nearest x2 + add
            ops.resize_nearest(lat[i], lat[i - 1], accumulate=True)
        outs = [k(lat[i]) for i, k in enumerate(self.k_out)]
        while len(outs) < self.num_outs:                            # fpn.py:126: max_pool2d(k=1, stride=2)
            p = outs[-1]
            n, h, w, c = p.shape
            q = empty_nhwc(n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c, p.dtype, p.device)
            ops.pool2d(p, q, 1, 2, 0)
            outs.append(q)
        return tuple(outs)


# ============================================================================ BFPTcea
class _LiteFlowNetCorr(nn.Module):
    def __init__(self, ch_in):
        super().__init__()

        def conv(a, b):
            return nn.Sequential(nn.Conv2d(a, b, 3, 1, 1, bias=True), nn.LeakyReLU(0.1, inplace=True))
        self.flow_estimator = nn.Module()
        self.flow_estimator.convs = nn.Sequential(conv(ch_in, 64), conv(64, 64), conv(64, 32),
                                                  nn.Conv2d(32, 2, 3, 1, 1, bias=True))


class _TCEAFusion(nn.Module):
    def __init__(self, nf, nframes):
        super().__init__()
        self.tAtt_1 = nn.Conv2d(nf, nf, 3, 1, 1)
        self.tAtt_2 = nn.Conv2d(nf, nf, 3, 1, 1)
        self.fea_fusion = nn.Conv2d(nframes * nf, nf, 1, 1)
        self.sAtt_1 = nn.Conv2d(nframes * nf, nf, 1, 1)
        self.sAtt_2 = nn.Conv2d(nf * 2, nf, 1, 1)
        self.sAtt_3 = nn.Conv2d(nf, nf, 3, 1, 1)
        self.sAtt_4 = nn.Conv2d(nf, nf, 3, 1, 1)
        self.sAtt_add_1 = nn.Conv2d(nf, nf, 1, 1)
        self.sAtt_add_2 = nn.Conv2d(nf, nf, 1, 1)


@EXTRA_NECKS.register_module
class BFPTcea(_Prepared):
    """mmdet/models/extra_necks/bfp_tcea.py:13-149 (refine_level 0, refine_type 'conv', 2 frames, center 0)."""

    def __init__(self, in_channels, num_levels, refine_level=1, refine_type=None, nframes=3, center=None,
                 stack_type='add', conv_cfg=None, norm_cfg=None):
        super().__init__()
        assert refine_level == 0 and refine_type == 'conv' and nframes == 2 and center == 0, \
            "only the fusetrack.py configuration is implemented"
        self.in_channels, self.num_levels = in_channels, num_levels
        self.liteflownet = _LiteFlowNetCorr(in_channels + 2 + 81)
        self.tcea_fusion = _TCEAFusion(in_channels, nframes)
        self.refine = _ConvModule(in_channels, in_channels, 3, 1)

    def _pack(self):
        fe = self.liteflownet.flow_estimator.convs
        self.k_flow = [_conv(fe[0][0], act=ACT_LRELU), _conv(fe[1][0], act=ACT_LRELU), _conv(fe[2][0], act=ACT_LRELU),
                       _conv(fe[3])]
        t = self.tcea_fusion
        self.k = dict(tAtt_1=_conv(t.tAtt_1), tAtt_2=_conv(t.tAtt_2), fea_fusion=_conv(t.fea_fusion, act=ACT_LRELU),
                      sAtt_1=_conv(t.sAtt_1, act=ACT_LRELU), sAtt_2=_conv(t.sAtt_2, act=ACT_LRELU),
                      sAtt_3=_conv(t.sAtt_3, act=ACT_LRELU), sAtt_4=_conv(t.sAtt_4),
                      sAtt_add_1=_conv(t.sAtt_add_1, act=ACT_LRELU), sAtt_add_2=_conv(t.sAtt_add_2),
                      refine=_conv(self.refine.conv, act=ACT_RELU))

    def forward(self, inputs, ref_inputs, flow_init, taps=None):
        """inputs/ref_inputs: tuples of NHWC pyramids; flow_init: NHWC fp32 [1,h,w,2] at level-0 size."""
        self.prepare()
        assert len(inputs) == self.num_levels
        x0 = inputs[0]
        n, h, w, c = x0.shape
        dt, dev = x0.dtype, x0.device
        # cat buffer of LiteFlowNetCorr: [bsf(256) | corr(81) | flow_init(2)] (flow_modules.py:67-70);
        # the gather writes bsf straight into its slice, the correlation into the next one.
        ccat = c + 81 + 2
        cat = empty_nhwc(n, h, w, ccat, dt, dev)
        bsf = cat[..., :c]
        br = ops.Branch("bfp_ref")                 # the reference frame's gather + warp next to the current frame's gather
        with br:
            ref_bsf = empty_nhwc(n, h, w, c, dt, dev)
            ops.bfp_gather(list(ref_inputs), ref_bsf)
            warp = empty_nhwc(n, h, w, c, dt, dev)
            ops.flow_warp(ref_bsf, flow_init, warp)
        ops.bfp_gather(list(inputs), bsf)
        br.join(warp, ref_bsf)
        ops.correlation(bsf, warp, cat[..., c:c + 81], 4, 4, 1, 1)
        ops.copy_scale(flow_init, cat[..., c + 81:c + 83])
        t = self.k_flow[0](cat)
        t = self.k_flow[1](t)
        t = self.k_flow[2](t)
        flow_fine = self.k_flow[3](t, out_dtype=torch.float32)
        warp2 = ref_bsf                                    # reuse
        ops.flow_warp(warp, flow_fine, warp2)
        k = self.k
        emb_ref = k['tAtt_2'](bsf)
        emb0 = k['tAtt_1'](bsf)
        emb1 = k['tAtt_1'](warp2)
        aligned = empty_nhwc(n, h, w, 2 * c, dt, dev)
        ops.tcea_temporal(bsf, warp2, emb0, emb1, emb_ref, aligned)
        fea = k['fea_fusion'](aligned)
        att = k['sAtt_1'](aligned)
        h2, w2 = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
        pcat = empty_nhwc(n, h2, w2, 2 * c, dt, dev)
        ops.pool2d(att, pcat[..., :c], 3, 2, 1, avg=False)
        ops.pool2d(att, pcat[..., c:], 3, 2, 1, avg=True)
        att = k['sAtt_3'](k['sAtt_2'](pcat))
        att_up = empty_nhwc(n, 2 * h2, 2 * w2, c, dt, dev)
        ops.resize_bilinear(att, att_up)
        att = k['sAtt_4'](att_up)
        att_add = k['sAtt_add_2'](k['sAtt_add_1'](att))
        fused = emb0                                        # reuse
        ops.tcea_combine(fea, att, att_add, fused)
        refined = k['refine'](fused)
        outs = []
        for i in range(self.num_levels):
            o = torch.empty_like(inputs[i])
            ops.bfp_scatter(refined, inputs[i], o)
            outs.append(o)
        if taps is not None:
            taps.update(bsf=bsf, warp_bsf=warp, flow_fine=flow_fine, warp_bsf2=warp2, refined=refined)
        return tuple(outs)


# ============================================================================ UPSNetFPN
class _DeformConv(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, 3, 3))
        stdv = 1.0 / math.sqrt(cin * 9)
        self.weight.data.uniform_(-stdv, stdv)


class _DeformConvWithOffset(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv_offset = nn.Conv2d(cin, 18, 3, 1, 1)
        self.conv = _DeformConv(cin, cout)


@PANOPTIC.register_module
class UPSNetFPN(_Prepared):
    """mmdet/models/panoptic/upsnetFPN.py:14-81."""

    def __init__(self, in_channels, out_channels, num_levels, num_things_classes, num_classes, ignore_label,
                 loss_weight, conv_cfg=None, norm_cfg=None):
        super().__init__()
        self.in_channels, self.out_channels, self.num_levels = in_channels, out_channels, num_levels
        self.num_things_classes, self.num_classes = num_things_classes, num_classes
        self.num_stuff_classes = num_classes - num_things_classes
        self.ignore_label, self.loss_weight = ignore_label, loss_weight
        self.deform_convs = nn.ModuleList([nn.Sequential(
            _DeformConvWithOffset(in_channels, in_channels), nn.GroupNorm(32, in_channels), nn.ReLU(inplace=True),
            _DeformConvWithOffset(in_channels, out_channels), nn.GroupNorm(32, out_channels), nn.ReLU(inplace=True),
            _DeformConvWithOffset(out_channels, out_channels), nn.GroupNorm(32, out_channels), nn.ReLU(inplace=True))])
        self.conv_pred = _ConvModule(out_channels * 4, num_classes, 1)
        # below this many pixels (< 1 tile per SM) the fused kernel is latency bound and im2col + GEMM is faster (measured)
        self.fused_dcn_min_pixels = 128 * 256

    def _pack(self):
        seq = self.deform_convs[0]
        self.k_dcn = []
        for i in (0, 3, 6):
            d, gn = seq[i], seq[i + 1]
            w = d.conv.weight.detach()
            co, ci = w.shape[:2]
            # columns are tap-major: k*C + c  (vps_deform_im2col) -> 1x1 conv weight [co, 9*ci]
            w1 = w.permute(0, 2, 3, 1).reshape(co, 9 * ci, 1, 1).contiguous()
            self.k_dcn.append(dict(off=_conv(d.conv_offset), gemm=Conv(w1, None), pk3=ops.PackedConv(w, None),
                                   gamma=gn.weight.detach().float().contiguous(),
                                   beta=gn.bias.detach().float().contiguous(), eps=gn.eps, groups=gn.num_groups))
        self.k_pred = _conv(self.conv_pred.conv)

    def _stack(self, x, out_last=None):
        n, h, w, _ = x.shape
        for j, L in enumerate(self.k_dcn):
            off = L['off'](x, out_dtype=torch.float32)
            if x.dtype == torch.bfloat16 and x.shape[3] % 64 == 0 and L['pk3'].cout <= 256 and n * h * w >= self.fused_dcn_min_pixels:
                # fused: sampled columns go straight into the tensor-core operand ring (no 9x column matrix in HBM)
                y = empty_nhwc(n, h, w, L['pk3'].cout, x.dtype, x.device)
                ops.deform_conv_tc(x, off, L['pk3'], y)
            elif ops.f32_tc_ok(x) and x.shape[3] % 32 == 0:
                # tc32 parity precision: same fusion with fp32 activations split into fp16 operand planes by the sampling warps
                y = empty_nhwc(n, h, w, L['pk3'].cout, x.dtype, x.device)
                ops.deform_conv_tc32(x, off, L['pk3'], y)
            else:
                cols = empty_nhwc(n, h, w, 9 * x.shape[3], x.dtype, x.device)
                ops.deform_im2col(x, off, cols)
                y = L['gemm'](cols)
            dst = out_last if (j == len(self.k_dcn) - 1 and out_last is not None) else y
            ops.groupnorm(y, dst, L['gamma'], L['beta'], L['groups'], L['eps'], relu=True)
            x = dst
        return x

    def forward(self, inputs, want_full=False):
        """returns (fcn_output or None, fcn_score NHWC fp32 [1,h,w,19])."""
        self.prepare()
        assert len(inputs) == self.num_levels
        n, h, w, _ = inputs[0].shape
        co = self.out_channels
        feat = empty_nhwc(n, h, w, co * self.num_levels, inputs[0].dtype, inputs[0].device)
        self._stack(inputs[0], out_last=feat[..., :co])
        for i in range(1, self.num_levels):
            p = self._stack(inputs[i])
            ops.resize_bilinear(p, feat[..., i * co:(i + 1) * co])       # upsnetFPN.py:74-76
        fcn_score = self.k_pred(feat, out_dtype=torch.float32)
        fcn_output = None
        if want_full:
            fcn_output = empty_nhwc(n, 4 * h, 4 * w, self.num_classes, torch.float32, feat.device)
            ops.resize_bilinear(fcn_score, fcn_output)
        return fcn_output, fcn_score


# ============================================================================ RPN
def _gen_base_anchors(base_size, scales, ratios):
    """anchor_generator.py:18-49 (scale_major, ctr=None) -- host-side constant table."""
    w = h = float(base_size)
    x_ctr, y_ctr = 0.5 * (w - 1), 0.5 * (h - 1)
    out = []
    for r in ratios:
        hr = math.sqrt(r)
        wr = 1.0 / hr
        for s in scales:
            ws, hs = w * wr * s, h * hr * s
            out.append([x_ctr - 0.5 * (ws - 1), y_ctr - 0.5 * (hs - 1), x_ctr + 0.5 * (ws - 1), y_ctr + 0.5 * (hs - 1)])
    # torch .round() = half to even on fp32 values
    t = torch.tensor(out, dtype=torch.float32)
    return torch.round(t)


@HEADS.register_module
class RPNHead(_Prepared):
    """mmdet/models/anchor_heads/rpn_head.py:12-104 + anchor_head.py:14-223 (sigmoid objectness)."""

    def __init__(self, in_channels, feat_channels=256, anchor_scales=[8, 16, 32], anchor_ratios=[0.5, 1.0, 2.0],
                 anchor_strides=[4, 8, 16, 32, 64], anchor_base_sizes=None, target_means=(.0, .0, .0, .0),
                 target_stds=(1.0, 1.0, 1.0, 1.0), loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.0)):
        super().__init__()
        self.in_channels, self.feat_channels = in_channels, feat_channels
        self.anchor_scales, self.anchor_ratios, self.anchor_strides = anchor_scales, anchor_ratios, list(anchor_strides)
        self.anchor_base_sizes = list(anchor_strides) if anchor_base_sizes is None else anchor_base_sizes
        self.target_means, self.target_stds = target_means, target_stds
        assert tuple(target_means) == (0, 0, 0, 0) and tuple(target_stds) == (1, 1, 1, 1)
        self.use_sigmoid_cls = loss_cls.get('use_sigmoid', False)
        assert self.use_sigmoid_cls
        self.loss_cls, self.loss_bbox = build_loss(loss_cls), build_loss(loss_bbox)
        self.num_anchors = len(anchor_ratios) * len(anchor_scales)
        self.rpn_conv = nn.Conv2d(in_channels, feat_channels, 3, padding=1)
        self.rpn_cls = nn.Conv2d(feat_channels, self.num_anchors, 1)
        self.rpn_reg = nn.Conv2d(feat_channels, self.num_anchors * 4, 1)

    def _pack(self):
        dev = self.rpn_conv.weight.device
        self.k_conv = _conv(self.rpn_conv, act=ACT_RELU)
        # sibling 1x1 heads fused into one GEMM: channels [0,A) = objectness, [A,5A) = deltas
        w = torch.cat([self.rpn_cls.weight, self.rpn_reg.weight], 0).detach()
        b = torch.cat([self.rpn_cls.bias, self.rpn_reg.bias], 0).detach()
        self.k_head = Conv(w, b)
        self.base_anchors = [_gen_base_anchors(s, self.anchor_scales, self.anchor_ratios).to(dev) for s in self.anchor_base_sizes]

    def forward(self, feats):
        """-> list of fused NHWC fp32 maps [1,h,w,5A] (cls | reg)."""
        self.prepare()
        return [self.k_head(self.k_conv(x), out_dtype=torch.float32) for x in feats]

    def get_bboxes(self, heads, img_shape, cfg, taps=None):
        """get_bboxes_single (rpn_head.py:55-104) for batch 1, all on device.
        Returns (proposals [max_num,5], rois [max_num,5], n_dev int32[1])."""
        A = self.num_anchors
        dev = heads[0].device
        nlev = len(heads)
        pre, post, max_num = cfg['nms_pre'], cfg['nms_post'], cfg['max_num']
        assert not cfg.get('nms_across_levels', False) and cfg.get('min_bbox_size', 0) == 0
        seg = min(pre, post) if pre > 0 else post
        dets_cat = torch.zeros(nlev * seg, 5, device=dev)
        counts = torch.zeros(nlev, dtype=torch.int32, device=dev)
        dets_all = torch.zeros(nlev * seg, 5, device=dev)          # level l: rows [l*seg, l*seg + ks[l])
        ks = []
        for l, hd in enumerate(heads):
            _, h, w, _ = hd.shape
            n = h * w * A
            scores = torch.empty(n, device=dev)
            ops.sigmoid_flat(hd[..., :A], scores)
            s_sorted = torch.empty(n, device=dev)
            i_sorted = torch.empty(n, dtype=torch.int32, device=dev)
            ws = torch.empty(ops.sort_ws_bytes(n), dtype=torch.uint8, device=dev)
            ops.sort_desc(scores, s_sorted, i_sorted, n, ws)
            k = min(n, pre) if pre > 0 else n
            assert k <= seg or pre <= 0
            k = min(k, seg)
            ks.append(k)
            ops.rpn_decode(s_sorted, i_sorted, k, hd[..., A:5 * A], self.anchor_strides[l], self.base_anchors[l],
                           float(img_shape[0]), float(img_shape[1]), dets_all[l * seg:l * seg + k])
        # the per-level NMS of get_bboxes_single, all levels in one launch pair
        keep = torch.empty(nlev * seg, dtype=torch.int32, device=dev)
        nws = torch.empty(max(nlev * ops.nms_ws_bytes(seg), 8), dtype=torch.uint8, device=dev)
        ops.nms_batch(dets_all, ks, seg, cfg['nms_thr'], keep, counts, nws)
        for l in range(nlev):
            ops.gather_rows(dets_all[l * seg:(l + 1) * seg], keep[l * seg:(l + 1) * seg], ks[l], 5,
                            dets_cat[l * seg:l * seg + ks[l]], n_dev=counts[l:l + 1])
        ntot = nlev * seg
        proposals = torch.empty(max_num, 5, device=dev)
        rois = torch.empty(max_num, 5, device=dev)
        total = torch.zeros(1, dtype=torch.int32, device=dev)
        ops.rpn_finalize(dets_cat, counts, nlev, seg, max_num, torch.empty(ntot, device=dev), torch.empty(ntot, device=dev),
                         torch.empty(ntot, dtype=torch.int32, device=dev),
                         torch.empty(ops.sort_ws_bytes(ntot), dtype=torch.uint8, device=dev), proposals, rois, total)
        if taps is not None:
            taps.update(rpn_dets_cat=dets_cat, rpn_counts=counts)
        return proposals, rois, total


# ============================================================================ RoI extractor / heads
@ROI_EXTRACTORS.register_module
class SingleRoIExtractor(nn.Module):
    """mmdet/models/roi_extractors/single_level.py:11-107 with roi_layer type RoIAlign (roi_align.py:59-87)."""

    def __init__(self, roi_layer, out_channels, featmap_strides, finest_scale=56):
        super().__init__()
        cfg = dict(roi_layer)
        assert cfg.pop('type') == 'RoIAlign', "only RoIAlign is on the FuseTrack path"
        self.out_size = cfg['out_size']
        self.sample_num = cfg.get('sample_num', 0)
        assert self.sample_num > 0 and finest_scale == 56
        self.out_channels, self.featmap_strides, self.finest_scale = out_channels, list(featmap_strides), finest_scale

    @property
    def num_inputs(self):
        return len(self.featmap_strides)

    def init_weights(self):
        pass

    def forward(self, feats, rois, nroi, nroi_dev=None, out=None):
        """feats: NHWC maps; rois: device f32 [>=nroi,5] -> NHWC [nroi, S, S, C]."""
        if out is None:
            out = empty_nhwc(nroi, self.out_size, self.out_size, self.out_channels, feats[0].dtype, feats[0].device)
        ops.roi_align(list(feats[:self.num_inputs]), self.featmap_strides, rois, nroi, out, self.sample_num, nroi_dev)
        return out


def _fc_from_roi_layout(weight, c, s):
    """FC columns (c,y,x) of the reference's flatten (convfc_bbox_head.py:143) -> (y,x,c) of the NHWC RoI features."""
    o = weight.shape[0]
    return weight.view(o, c, s, s).permute(0, 2, 3, 1).reshape(o, s * s * c).contiguous()


@HEADS.register_module
class SharedFCBBoxHead(_Prepared):
    """mmdet/models/bbox_heads/convfc_bbox_head.py:171-185 (-> ConvFCBBoxHead 8-168, BBoxHead bbox_head.py:14-79)."""

    def __init__(self, num_fcs=2, fc_out_channels=1024, with_avg_pool=False, with_cls=True, with_reg=True, roi_feat_size=7,
                 in_channels=256, num_classes=81, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
                 reg_class_agnostic=False, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0)):
        super().__init__()
        assert num_fcs >= 1 and not with_avg_pool and with_cls and with_reg and not reg_class_agnostic
        self.in_channels, self.roi_feat_size, self.num_classes = in_channels, roi_feat_size, num_classes
        self.target_means, self.target_stds = target_means, target_stds
        self.loss_cls, self.loss_bbox = build_loss(loss_cls), build_loss(loss_bbox)
        dims = [in_channels * roi_feat_size * roi_feat_size] + [fc_out_channels] * num_fcs
        self.shared_fcs = nn.ModuleList([nn.Linear(dims[i], dims[i + 1]) for i in range(num_fcs)])
        self.fc_cls = nn.Linear(fc_out_channels, num_classes)
        self.fc_reg = nn.Linear(fc_out_channels, 4 * num_classes)

    def _pack(self):
        fcs = []
        for i, fc in enumerate(self.shared_fcs):
            w = fc.weight.detach()
            if i == 0:
                w = _fc_from_roi_layout(w, self.in_channels, self.roi_feat_size)
            fcs.append(Linear(w, fc.bias.detach(), act=ACT_RELU))
        self.k_fcs = fcs
        self.k_out = Linear(torch.cat([self.fc_cls.weight, self.fc_reg.weight], 0).detach(),
                            torch.cat([self.fc_cls.bias, self.fc_reg.bias], 0).detach())

    def forward(self, roi_feats):
        """roi_feats NHWC [n,7,7,C] -> (cls_score [n,9], bbox_pred [n,36]) fp32 device tensors."""
        self.prepare()
        n = roi_feats.shape[0]
        x = roi_feats.reshape(n, -1)
        for fc in self.k_fcs:
            x = fc(x)
        y = self.k_out(x, out_dtype=torch.float32)
        nc = self.num_classes
        return y[:, :nc], y[:, nc:5 * nc], y


@HEADS.register_module
class TrackHead(_Prepared):
    """mmdet/models/track_heads/track_head.py:20-174."""

    def __init__(self, with_avg_pool=False, num_fcs=2, in_channels=256, roi_feat_size=7, fc_out_channels=1024,
                 match_coeff=None, bbox_dummy_iou=0, dynamic=True,
                 loss_match=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)):
        super().__init__()
        assert not with_avg_pool and dynamic and bbox_dummy_iou == 0
        self.in_channels, self.roi_feat_size, self.match_coeff = in_channels, roi_feat_size, match_coeff
        self.fc_out_channels = fc_out_channels
        dims = [in_channels * roi_feat_size * roi_feat_size] + [fc_out_channels] * num_fcs
        self.fcs = nn.ModuleList([nn.Linear(dims[i], dims[i + 1]) for i in range(num_fcs)])
        self.loss_match = build_loss(loss_match)

    def _pack(self):
        ks = []
        for i, fc in enumerate(self.fcs):
            w = fc.weight.detach()
            if i == 0:
                w = _fc_from_roi_layout(w, self.in_channels, self.roi_feat_size)
            ks.append(Linear(w, fc.bias.detach(), act=ACT_RELU if i < len(self.fcs) - 1 else ACT_NONE))
        self.k_fcs = ks

    def embed(self, roi_feats):
        """track_head.py:105-113: FC stack, ReLU between; -> fp32 [n, fc_out]."""
        self.prepare()
        x = roi_feats.reshape(roi_feats.shape[0], -1)
        for i, fc in enumerate(self.k_fcs):
            x = fc(x, out_dtype=torch.float32 if i == len(self.k_fcs) - 1 else None)
        return x


@HEADS.register_module
class FCNMaskHead(_Prepared):
    """mmdet/models/mask_heads/fcn_mask_head.py:14-103 (deconv upsampling)."""

    def __init__(self, num_convs=4, roi_feat_size=14, in_channels=256, conv_kernel_size=3, conv_out_channels=256,
                 upsample_method='deconv', upsample_ratio=2, num_classes=81, class_agnostic=False, conv_cfg=None,
                 norm_cfg=None, loss_mask=dict(type='CrossEntropyLoss', use_mask=True, loss_weight=1.0)):
        super().__init__()
        assert upsample_method == 'deconv' and upsample_ratio == 2 and not class_agnostic and norm_cfg is None
        self.num_classes = num_classes
        self.loss_mask = build_loss(loss_mask)
        self.convs = nn.ModuleList([_ConvModule(in_channels if i == 0 else conv_out_channels, conv_out_channels,
                                                conv_kernel_size, (conv_kernel_size - 1) // 2) for i in range(num_convs)])
        self.upsample = nn.ConvTranspose2d(conv_out_channels, conv_out_channels, 2, stride=2)
        self.conv_logits = nn.Conv2d(conv_out_channels, num_classes, 1)

    def _pack(self):
        self.k_convs = [_conv(m.conv, act=ACT_RELU) for m in self.convs]
        self.k_up = deconv2x2_s2(self.upsample.weight.detach(), self.upsample.bias.detach())
        self.k_logits = _conv(self.conv_logits)

    def forward(self, x):
        """x NHWC [k,14,14,C] -> NHWC fp32 [k,28,28,num_classes]."""
        self.prepare()
        for c in self.k_convs:
            x = c(x)
        n, h, w, _ = x.shape
        y = empty_nhwc(n, 2 * h, 2 * w, self.upsample.out_channels, x.dtype, x.device)
        self.k_up(x, y, act=ACT_RELU)
        return self.k_logits(y, out_dtype=torch.float32)
