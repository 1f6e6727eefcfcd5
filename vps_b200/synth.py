"""Deterministic synthetic weight sets for any module tree with the reference's PanopticFuseTrack state_dict
layout (the oracle model and the vps_b200 detector share it).  There are no trained checkpoints offline
(download_weights.sh needs the network); these sets exercise every code path (SURVEY.md 8d):

  "A": the reference's init rules (kaiming / xavier / normal as cited in SURVEY A.13).  bn3.gamma = 0
       and score_thresh 0.6 mean residual branches vanish and nothing is detected -> plumbing only.
  "B": dense-random: every conv/linear kaiming-uniform-ish, BN gamma~U(.5,1.5), beta~N(0,.1), running
       stats random, non-zero DCN offsets, FlowNet2 xavier with small biases.
  "C": B + detection forcing: bbox_head.fc_cls scaled up / fc_reg scaled down so that dozens of RoIs pass
       the 0.6 threshold and the mask / tracking / fusion stages see real instances.

Pure parameter initialisation (torch RNG on CPU tensors); nothing here runs on the inference path.
"""
import math

import torch
import torch.nn as nn


def _kaiming_uniform(w, gain=1.0):
    fan_in = w[0].numel()
    bound = gain * math.sqrt(3.0 / fan_in)
    w.uniform_(-bound, bound)


@torch.no_grad()
def init_weights(model, kind="C", seed=0):
    g = torch.Generator().manual_seed(seed)

    def U(t, a, b):
        t.copy_(torch.rand(t.shape, generator=g) * (b - a) + a)

    def N(t, mean, std):
        t.copy_(torch.randn(t.shape, generator=g) * std + mean)

    if kind == "A":
        for name, m in model.named_modules():
            if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d, nn.Linear)):
                if name.startswith("flownet2"):
                    fan_in = m.weight[0].numel() if not isinstance(m, nn.ConvTranspose2d) else m.weight.shape[0] * m.weight[0, 0].numel()
                    fan_out = m.weight.shape[0] * m.weight[0, 0].numel() if not isinstance(m, nn.ConvTranspose2d) else m.weight[0].numel()
                    b = math.sqrt(6.0 / (fan_in + fan_out))
                    U(m.weight, -b, b)
                    if m.bias is not None:
                        U(m.bias, 0, 1)
                elif name.startswith("backbone"):
                    fan_out = m.weight.shape[0] * m.weight[0, 0].numel()
                    N(m.weight, 0, math.sqrt(2.0 / fan_out))
                elif name.startswith(("rpn_head", "track_head")):
                    N(m.weight, 0, 0.01); m.bias.zero_()
                elif name == "bbox_head.fc_cls":
                    N(m.weight, 0, 0.01); m.bias.zero_()
                elif name == "bbox_head.fc_reg":
                    N(m.weight, 0, 0.001); m.bias.zero_()
                else:   # xavier uniform (FPN, BFPTcea, UPSNetFPN, shared fcs); kaiming for mask head is close enough
                    fan_in = m.weight[0].numel()
                    fan_out = m.weight.shape[0] * (m.weight[0, 0].numel() if m.weight.dim() > 2 else 1)
                    b = math.sqrt(6.0 / (fan_in + fan_out))
                    U(m.weight, -b, b)
                    if m.bias is not None:
                        m.bias.zero_()
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.fill_(1); m.bias.zero_(); m.running_mean.zero_(); m.running_var.fill_(1)
                if name.endswith("bn3"):
                    m.weight.zero_()
            elif m.__class__.__name__ in ("DeformConv", "_DeformConv"):
                # the reference's DeformConv.reset_parameters (uniform +-1/sqrt(fan_in)), drawn from the seeded generator:
                # left to the constructor, these weights came from the global RNG and changed with whatever ran before
                stdv = 1.0 / math.sqrt(m.weight[0].numel())
                U(m.weight, -stdv, stdv)
        return model

    for name, m in model.named_modules():
        if isinstance(m, (nn.Conv2d, nn.Linear)):
            _g = 1.4 if not name.startswith("flownet2") else 1.0
            fan_in = m.weight[0].numel()
            bound = _g * math.sqrt(3.0 / fan_in)
            U(m.weight, -bound, bound)
            if m.bias is not None:
                N(m.bias, 0, 0.05)
        elif isinstance(m, nn.ConvTranspose2d):
            fan_in = m.weight.shape[0] * m.weight[0, 0].numel() / 4.0   # stride-2: ~1/4 of taps hit each output
            bound = math.sqrt(3.0 / fan_in)
            U(m.weight, -bound, bound)
            if m.bias is not None:
                N(m.bias, 0, 0.05)
        elif isinstance(m, nn.BatchNorm2d):
            U(m.weight, 0.5, 1.5); N(m.bias, 0, 0.1); N(m.running_mean, 0, 0.1); U(m.running_var, 0.5, 1.5)
            if name.endswith("bn3"):
                m.weight.mul_(0.5)      # keep the residual trunk from blowing up over 16 blocks
        elif isinstance(m, nn.GroupNorm):
            U(m.weight, 0.5, 1.5); N(m.bias, 0, 0.1)
        elif m.__class__.__name__ in ("DeformConv", "_DeformConv"):
            fan_in = m.weight[0].numel()
            bound = 1.4 * math.sqrt(3.0 / fan_in)
            U(m.weight, -bound, bound)
    # DCN offsets: moderate non-zero offsets (a few pixels)
    for name, m in model.named_modules():
        if name.endswith("conv_offset"):
            N(m.weight, 0, 0.02); N(m.bias, 0, 0.5)
    # FlowNet2 predicts flows through 5 stacked nets; keep predictions O(1 px)
    for name, m in model.named_modules():
        if name.startswith("flownet2") and "predict_flow" in name:
            m.weight.mul_(0.2)
    # RPN: spread objectness and keep deltas moderate
    model.rpn_head.rpn_cls.weight.mul_(2.0)
    model.rpn_head.rpn_reg.weight.mul_(0.3)
    if kind == "C":
        model.bbox_head.fc_cls.weight.mul_(6.0)
        model.bbox_head.fc_cls.bias[0] -= 1.0
        model.bbox_head.fc_reg.weight.mul_(0.3)
        model.mask_head.conv_logits.weight.mul_(3.0)
    return model




# LSUV-style output-layer rescaling of weight set ("C", seed 0): the factors oracle/weights.calibrate() measures on
# its fixed 128x256 calibration pair (O(1) pyramid features, ~1.5 px flows, un-saturated class scores, O(1) mask
# logits / tracker scores).  Stored as a table so the product side needs no forward passes and no oracle import;
# tests/test_boundary.py::test_synth_table_matches_oracle_calibration keeps it in sync.
CALIB_C0 = {
    "neck.lateral_convs.0.conv": 0.1340239941767244,
    "neck.lateral_convs.1.conv": 0.06618518382065915,
    "neck.lateral_convs.2.conv": 0.020061241463040818,
    "neck.lateral_convs.3.conv": 0.00988386385144237,
    "neck.fpn_convs.0.conv": 0.37838611009767953,
    "neck.fpn_convs.1.conv": 0.44232100248994954,
    "neck.fpn_convs.2.conv": 0.584843754806467,
    "neck.fpn_convs.3.conv": 0.813946068310941,
    "extra_neck.liteflownet.flow_estimator.convs.3": 1.5344217999474192,
    "extra_neck.tcea_fusion.tAtt_1": 0.3559170067085267,
    "extra_neck.tcea_fusion.tAtt_2": 0.32918161154036085,
    "extra_neck.tcea_fusion.sAtt_4": 1.1613397598588795,
    "extra_neck.refine.conv": 0.7676233052990034,
    "panopticFPN.conv_pred.conv": 1.6510677332501664,
    "rpn_head.rpn_cls": 0.2886631487937804,
    "rpn_head.rpn_reg": 0.6935749642411232,
    "bbox_head.shared_fcs.0": 0.7816216349618003,
    "bbox_head.shared_fcs.1": 1.014483690296394,
    "bbox_head.fc_cls": 0.5192481280262087,
    "bbox_head.fc_reg": 1.342059493296237,
    "track_head.fcs.0": 0.8488115668424713,
    "track_head.fcs.1": 0.042735997588443764,
    "mask_head.conv_logits": 0.6610493053140023,
    "flownet2.flownetfusion.predict_flow0": 26.286098491233904
}


@torch.no_grad()
def make_weights(model, kind="C", seed=0, calibrated=True):
    """Initialise `model` in place with the synthetic weight set; returns the model."""
    init_weights(model, kind, seed)
    if calibrated:
        if not (kind == "C" and seed == 0):
            raise ValueError("calibration table only exists for weight set ('C', 0)")
        mods = dict(model.named_modules())
        for name, s in CALIB_C0.items():
            m = mods[name]
            m.weight.mul_(s)
            if getattr(m, "bias", None) is not None:
                m.bias.mul_(s)
    return model
