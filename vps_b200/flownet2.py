"""vps_b200 FlowNet2 (frozen optical-flow sub-network of PanopticFuseTrack).

Mirrors mmdet/models/flow_modules/{flownet2.py:32-198, FlowNetC.py:13-128, FlowNetS.py:15-94,
FlowNetSD.py:11-106, FlowNetFusion.py:11-67, submodules.py:7-38}: same sub-module and parameter names
(`flownetc.conv1.0.weight`, `flownets_1.deconv5.0.weight`, ...), inference (eval) dataflow only.

Design points: every torch.cat of the reference is a pre-allocated NHWC concat buffer whose
producers write their channel slice directly (conv epilogues, transposed-conv phase kernels, the
correlation kernel); ConvTranspose2d(4,2,1) runs as four stride-phase 2x2 convolutions on the
tensor-core kernel; `x*div_flow`, `x/div_flow` scalings are folded into the resize kernels; warping
flows are kept in fp32 regardless of the activation dtype.
"""
import torch
import torch.nn as nn

from . import ops
from .layers import ACT_LRELU, ACT_NONE, Conv, StemConv7x7s2, deconv4x4_s2, empty_nhwc
from .modules import _Prepared, _conv


def _c(cin, cout, k=3, s=1):
    return nn.Sequential(nn.Conv2d(cin, cout, k, s, (k - 1) // 2, bias=True), nn.LeakyReLU(0.1, inplace=True))


def _ic(cin, cout):
    return nn.Sequential(nn.Conv2d(cin, cout, 3, 1, 1, bias=True))


def _pf(cin):
    return nn.Conv2d(cin, 2, 3, 1, 1, bias=True)


def _dc(cin, cout):
    return nn.Sequential(nn.ConvTranspose2d(cin, cout, 4, 2, 1, bias=True), nn.LeakyReLU(0.1, inplace=True))


class _Net(nn.Module):
    """parameter holder + packed kernels of one FlowNet sub-network"""

    def pack(self):
        self.k = {}
        for name, m in self.named_children():
            if isinstance(m, nn.Sequential) and isinstance(m[0], nn.ConvTranspose2d):
                self.k[name] = deconv4x4_s2(m[0].weight.detach(), None if m[0].bias is None else m[0].bias.detach())
            elif isinstance(m, nn.Sequential) and m[0].kernel_size == (7, 7) and m[0].stride == (2, 2):
                self.k[name] = StemConv7x7s2(m[0].weight.detach(), m[0].bias.detach(), act=ACT_LRELU)
            elif isinstance(m, nn.Sequential):
                self.k[name] = _conv(m[0], act=ACT_LRELU if len(m) > 1 else ACT_NONE)
            elif isinstance(m, nn.ConvTranspose2d):      # 2->2 flow up-sampler: dedicated kernel, weights as arguments
                wl = m.weight.detach().float().cpu().reshape(-1).tolist()
                bl = None if m.bias is None else m.bias.detach().float().cpu().tolist()
                self.k[name] = (lambda x, y, wl=wl, bl=bl: ops.flow_deconv(x, wl, bl, y))
            elif isinstance(m, nn.Conv2d):
                self.k[name] = _conv(m)

    @staticmethod
    def _buf(like, h, w, c):
        return empty_nhwc(like.shape[0], h, w, c, like.dtype, like.device)

    def _refine(self, feats, c6, inter=False):
        """Decoder shared by FlowNetC/S (raw concat -> predict) and FlowNetSD (inter_conv -> predict).
        feats = [c2, c3, c4, c5] encoder maps ALREADY living in channel slice [0:Ci) of their concat buffer;
        returns flow2 (fp32)."""
        k = self.k
        cur = c6
        flow = k['predict_flow6'](cur)
        for lvl in (5, 4, 3, 2):
            cat, c_enc, c_dec = feats[lvl]
            _, h, w, _ = cat.shape
            k['deconv%d' % lvl](cur, cat[..., c_enc:c_enc + c_dec], act=ACT_LRELU)
            k['upsampled_flow%d_to_%d' % (lvl + 1, lvl)](flow, cat[..., c_enc + c_dec:c_enc + c_dec + 2])
            src = k['inter_conv%d' % lvl](cat) if inter else cat
            last = lvl == 2
            flow = k['predict_flow%d' % lvl](src, out_dtype=torch.float32 if last else None)
            cur = cat
        return flow


class _FlowNetC(_Net):
    def __init__(self):
        super().__init__()
        self.conv1, self.conv2, self.conv3 = _c(3, 64, 7, 2), _c(64, 128, 5, 2), _c(128, 256, 5, 2)
        self.conv_redir = _c(256, 32, 1, 1)
        self.conv3_1 = _c(473, 256)
        self.conv4, self.conv4_1 = _c(256, 512, 3, 2), _c(512, 512)
        self.conv5, self.conv5_1 = _c(512, 512, 3, 2), _c(512, 512)
        self.conv6, self.conv6_1 = _c(512, 1024, 3, 2), _c(1024, 1024)
        self.deconv5, self.deconv4, self.deconv3, self.deconv2 = _dc(1024, 512), _dc(1026, 256), _dc(770, 128), _dc(386, 64)
        self.predict_flow6, self.predict_flow5, self.predict_flow4 = _pf(1024), _pf(1026), _pf(770)
        self.predict_flow3, self.predict_flow2 = _pf(386), _pf(194)
        for a, b in ((6, 5), (5, 4), (4, 3), (3, 2)):
            setattr(self, 'upsampled_flow%d_to_%d' % (a, b), nn.ConvTranspose2d(2, 2, 4, 2, 1, bias=True))

    def forward(self, x6):
        """x6: NHWC [1,H,W,6] (img0 | img1) -> flow2 fp32 NHWC [1,H/4,W/4,2] (FlowNetC.py:71-128)."""
        k = self.k
        n, H, W, _ = x6.shape
        B = lambda h, w, c: self._buf(x6, h, w, c)
        cat2 = B(H // 4, W // 4, 194); cat3 = B(H // 8, W // 8, 386)
        cat4 = B(H // 16, W // 16, 770); cat5 = B(H // 32, W // 32, 1026)
        c1a = k['conv1'](x6[..., 0:3]); c2a = k['conv2'](c1a, cat2[..., :128]); c3a = k['conv3'](c2a)
        c1b = k['conv1'](x6[..., 3:6]); c2b = k['conv2'](c1b); c3b = k['conv3'](c2b)
        in31 = B(H // 8, W // 8, 473)                      # cat(conv_redir 32, corr 441) FlowNetC.py:90
        k['conv_redir'](c3a, in31[..., :32])
        ops.correlation(c3a, c3b, in31[..., 32:473], 20, 20, 1, 2, act=ACT_LRELU, slope=0.1)
        k['conv3_1'](in31, cat3[..., :256])
        k['conv4_1'](k['conv4'](cat3[..., :256]), cat4[..., :512])
        k['conv5_1'](k['conv5'](cat4[..., :512]), cat5[..., :512])
        c6 = k['conv6_1'](k['conv6'](cat5[..., :512]))
        return self._refine({5: (cat5, 512, 512), 4: (cat4, 512, 256), 3: (cat3, 256, 128), 2: (cat2, 128, 64)}, c6)


class _FlowNetS(_Net):
    def __init__(self, cin=12):
        super().__init__()
        self.conv1, self.conv2, self.conv3 = _c(cin, 64, 7, 2), _c(64, 128, 5, 2), _c(128, 256, 5, 2)
        self.conv3_1 = _c(256, 256)
        self.conv4, self.conv4_1 = _c(256, 512, 3, 2), _c(512, 512)
        self.conv5, self.conv5_1 = _c(512, 512, 3, 2), _c(512, 512)
        self.conv6, self.conv6_1 = _c(512, 1024, 3, 2), _c(1024, 1024)
        self.deconv5, self.deconv4, self.deconv3, self.deconv2 = _dc(1024, 512), _dc(1026, 256), _dc(770, 128), _dc(386, 64)
        self.predict_flow6, self.predict_flow5, self.predict_flow4 = _pf(1024), _pf(1026), _pf(770)
        self.predict_flow3, self.predict_flow2 = _pf(386), _pf(194)
        for a, b in ((6, 5), (5, 4), (4, 3), (3, 2)):
            setattr(self, 'upsampled_flow%d_to_%d' % (a, b), nn.ConvTranspose2d(2, 2, 4, 2, 1, bias=False))

    def forward(self, x12):
        k = self.k
        n, H, W, _ = x12.shape
        B = lambda h, w, c: self._buf(x12, h, w, c)
        cat2 = B(H // 4, W // 4, 194); cat3 = B(H // 8, W // 8, 386)
        cat4 = B(H // 16, W // 16, 770); cat5 = B(H // 32, W // 32, 1026)
        k['conv2'](k['conv1'](x12), cat2[..., :128])
        k['conv3_1'](k['conv3'](cat2[..., :128]), cat3[..., :256])
        k['conv4_1'](k['conv4'](cat3[..., :256]), cat4[..., :512])
        k['conv5_1'](k['conv5'](cat4[..., :512]), cat5[..., :512])
        c6 = k['conv6_1'](k['conv6'](cat5[..., :512]))
        return self._refine({5: (cat5, 512, 512), 4: (cat4, 512, 256), 3: (cat3, 256, 128), 2: (cat2, 128, 64)}, c6)


class _FlowNetSD(_Net):
    def __init__(self):
        super().__init__()
        self.conv0 = _c(6, 64)
        self.conv1, self.conv1_1 = _c(64, 64, 3, 2), _c(64, 128)
        self.conv2, self.conv2_1 = _c(128, 128, 3, 2), _c(128, 128)
        self.conv3, self.conv3_1 = _c(128, 256, 3, 2), _c(256, 256)
        self.conv4, self.conv4_1 = _c(256, 512, 3, 2), _c(512, 512)
        self.conv5, self.conv5_1 = _c(512, 512, 3, 2), _c(512, 512)
        self.conv6, self.conv6_1 = _c(512, 1024, 3, 2), _c(1024, 1024)
        self.deconv5, self.deconv4, self.deconv3, self.deconv2 = _dc(1024, 512), _dc(1026, 256), _dc(770, 128), _dc(386, 64)
        self.inter_conv5, self.inter_conv4, self.inter_conv3, self.inter_conv2 = _ic(1026, 512), _ic(770, 256), _ic(386, 128), _ic(194, 64)
        self.predict_flow6, self.predict_flow5, self.predict_flow4 = _pf(1024), _pf(512), _pf(256)
        self.predict_flow3, self.predict_flow2 = _pf(128), _pf(64)
        for a, b in ((6, 5), (5, 4), (4, 3), (3, 2)):
            setattr(self, 'upsampled_flow%d_to_%d' % (a, b), nn.ConvTranspose2d(2, 2, 4, 2, 1))

    def forward(self, x6):
        k = self.k
        n, H, W, _ = x6.shape
        B = lambda h, w, c: self._buf(x6, h, w, c)
        cat2 = B(H // 4, W // 4, 194); cat3 = B(H // 8, W // 8, 386)
        cat4 = B(H // 16, W // 16, 770); cat5 = B(H // 32, W // 32, 1026)
        c1 = k['conv1_1'](k['conv1'](k['conv0'](x6)))
        k['conv2_1'](k['conv2'](c1), cat2[..., :128])
        k['conv3_1'](k['conv3'](cat2[..., :128]), cat3[..., :256])
        k['conv4_1'](k['conv4'](cat3[..., :256]), cat4[..., :512])
        k['conv5_1'](k['conv5'](cat4[..., :512]), cat5[..., :512])
        c6 = k['conv6_1'](k['conv6'](cat5[..., :512]))
        return self._refine({5: (cat5, 512, 512), 4: (cat4, 512, 256), 3: (cat3, 256, 128), 2: (cat2, 128, 64)}, c6,
                            inter=True)


class _FlowNetFusion(_Net):
    def __init__(self):
        super().__init__()
        self.conv0 = _c(11, 64)
        self.conv1, self.conv1_1 = _c(64, 64, 3, 2), _c(64, 128)
        self.conv2, self.conv2_1 = _c(128, 128, 3, 2), _c(128, 128)
        self.deconv1, self.deconv0 = _dc(128, 32), _dc(162, 16)
        self.inter_conv1, self.inter_conv0 = _ic(162, 32), _ic(82, 16)
        self.predict_flow2, self.predict_flow1, self.predict_flow0 = _pf(128), _pf(32), _pf(16)
        self.upsampled_flow2_to_1 = nn.ConvTranspose2d(2, 2, 4, 2, 1)
        self.upsampled_flow1_to_0 = nn.ConvTranspose2d(2, 2, 4, 2, 1)

    def forward(self, x11):
        k = self.k
        n, H, W, _ = x11.shape
        B = lambda h, w, c: self._buf(x11, h, w, c)
        cat0 = B(H, W, 82); cat1 = B(H // 2, W // 2, 162)
        k['conv0'](x11, cat0[..., :64])
        k['conv1_1'](k['conv1'](cat0[..., :64]), cat1[..., :128])
        c2 = k['conv2_1'](k['conv2'](cat1[..., :128]))
        flow2 = k['predict_flow2'](c2)
        k['deconv1'](c2, cat1[..., 128:160], act=ACT_LRELU)
        k['upsampled_flow2_to_1'](flow2, cat1[..., 160:162])
        flow1 = k['predict_flow1'](k['inter_conv1'](cat1))
        k['deconv0'](cat1, cat0[..., 64:80], act=ACT_LRELU)
        k['upsampled_flow1_to_0'](flow1, cat0[..., 80:82])
        return k['predict_flow0'](k['inter_conv0'](cat0), out_dtype=torch.float32)


class FlowNet2(_Prepared):
    """flownet2.py:32-198 with args.rgb_max = 255, fp16 = False, div_flow = 20."""

    def __init__(self, rgb_max=255.0, div_flow=20.0):
        super().__init__()
        self.rgb_max, self.div_flow = rgb_max, div_flow
        self.fused_glue = True       # build the inter-network concat inputs with one kernel each (ops.flownet_stage / flownet_cat3)
        self.flownetc = _FlowNetC()
        self.flownets_1 = _FlowNetS()
        self.flownets_2 = _FlowNetS()
        self.flownets_d = _FlowNetSD()
        self.flownetfusion = _FlowNetFusion()
        for p in self.parameters():
            p.requires_grad = False

    def _pack(self):
        for m in (self.flownetc, self.flownets_1, self.flownets_2, self.flownets_d, self.flownetfusion):
            m.pack()

    def forward(self, x6, taps=None):
        """x6: NHWC [1,H,W,6] = ((rgb - mean)/255 of img0 | img1) -> flow fp32 NHWC [1,H,W,2]."""
        self.prepare()
        n, H, W, _ = x6.shape
        dt, dev = x6.dtype, x6.device
        img0, img1 = x6[..., 0:3], x6[..., 3:6]
        f32 = lambda c: torch.empty(n, H, W, c, dtype=torch.float32, device=dev)

        def stage(flow2):
            """concat(x, resampled_img1, flow/div_flow, norm_diff) (flownet2.py:142-153) for FlowNetS."""
            cat = empty_nhwc(n, H, W, 12, dt, dev)
            if self.fused_glue:      # one kernel builds the 12-channel pixel (bit-identical to the five ops below)
                return ops.flownet_stage(x6, flow2, self.div_flow, 1.0 / self.div_flow, cat)
            flow = f32(2)
            ops.resize_bilinear(flow2, flow, mul=self.div_flow)       # upsample(flow2 * div_flow)
            ops.copy_scale(x6, cat[..., 0:6])
            ops.resample2d(img1, flow, cat[..., 6:9])
            ops.copy_scale(flow, cat[..., 9:11], 1.0 / self.div_flow)
            ops.channelnorm(img0, cat[..., 11:12], b=cat[..., 6:9])
            return cat

        # FlowNetSD only reads x6: parallel branch next to the FlowNetC -> S1 -> S2 chain
        br = ops.Branch("flownet_sd")
        with br:
            sd_flow2 = self.flownets_d(x6)
        c_flow2 = self.flownetc(x6)
        cat1 = stage(c_flow2)
        s1_flow2 = self.flownets_1(cat1)
        cat2 = stage(s1_flow2)
        s2_flow2 = self.flownets_2(cat2)
        br.join(sd_flow2)

        # concat3 = (img0, sd_flow, s2_flow, |sd_flow|, |s2_flow|, |img0 - warp_sd|, |img0 - warp_s2|) flownet2.py:189
        cat3 = empty_nhwc(n, H, W, 11, dt, dev)
        if self.fused_glue:
            ops.flownet_cat3(x6, s2_flow2, sd_flow2, self.div_flow, 1.0 / self.div_flow, cat3)
            out = self.flownetfusion(cat3)
            if taps is not None:
                taps.update(c_flow2=c_flow2, s1_flow2=s1_flow2, s2_flow2=s2_flow2, sd_flow2=sd_flow2, concat1=cat1, concat3=cat3)
            return out
        s2_flow, sd_flow = f32(2), f32(2)
        ops.resize_nearest(s2_flow2, s2_flow, mul=self.div_flow)          # upsample4(flow2 * div_flow)
        ops.resize_nearest(sd_flow2, sd_flow, mul=1.0 / self.div_flow)    # upsample3(flow2 / div_flow)
        ops.copy_scale(img0, cat3[..., 0:3])
        ops.copy_scale(sd_flow, cat3[..., 3:5])
        ops.copy_scale(s2_flow, cat3[..., 5:7])
        ops.channelnorm(sd_flow, cat3[..., 7:8])
        ops.channelnorm(s2_flow, cat3[..., 8:9])
        warped = empty_nhwc(n, H, W, 3, dt, dev)
        ops.resample2d(img1, sd_flow, warped)
        ops.channelnorm(img0, cat3[..., 9:10], b=warped)
        ops.resample2d(img1, s2_flow, warped)
        ops.channelnorm(img0, cat3[..., 10:11], b=warped)
        out = self.flownetfusion(cat3)
        if taps is not None:
            taps.update(c_flow2=c_flow2, s1_flow2=s1_flow2, s2_flow2=s2_flow2, sd_flow2=sd_flow2, concat1=cat1,
                        concat3=cat3)
        return out
