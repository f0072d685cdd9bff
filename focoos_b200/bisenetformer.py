"""BisenetFormer (real-time semantic segmenter) — host-side mirror of `focoos/models/bisenetformer/modelling.py` and
`focoos/nn/backbone/stdc.py` (SURVEY §8 rows a18-a19).  Parameter containers under the reference's state_dict keys
(505 entries for bisenetformer-l-ade) + `BisenetEngine`, a fused NHWC graph:

  * STDC backbone: ConvX = conv + folded BN + ReLU in one kernel; CatBottleneck is CONCAT-FREE — every branch writes its channel
    slice of the block's output buffer (widths C/2, C/4, C/8, C/8) and the next 3x3 conv reads that slice in place; stride-2 blocks
    use the depthwise 3x3/s2 + BN kernel and the 3x3/s2 average-pool skip (nn/backbone/stdc.py:153-172),
  * context path: ARM = 1x1 proj -> 3x3 ConvBNReLU -> global average pool -> 1x1 + BN + sigmoid gate (a [B,C] GEMM with the
    sigmoid in its epilogue) -> one gating kernel that also adds the global-context vector / the upsampled coarser level
    (bisenetformer/modelling.py:159-210),
  * spatial path + FFM: proj1(res3) + proj2(cp8) as one conv with the other as residual, 1x1 ConvBNReLU, gate, `feat*att + feat`
    in the gating kernel, conv_out (:224-235,266),
  * the 2-level masked transformer decoder, head and x8 sigmoid+bilinear upsample shared with the MaskFormer family.
"""
from __future__ import annotations

from dataclasses import dataclass, field, fields
from typing import List, Optional

import torch
import torch.nn as nn

from . import ops
from .engine import _packed_layers, _unpair
from .fai_mf import MaskFormerModelOutput, MFEngine, MultiScaleMaskedTransformerDecoder, _SegmentationModel
from .ports import ModelOutput, STDCConfig
from .trunks import STDC, ConvX, build_trunk, pack_trunk


@dataclass
class BisenetFormerConfig:
    """models/bisenetformer/config.py (fields of the registry JSON)."""

    backbone_config: STDCConfig = field(default_factory=STDCConfig)
    num_classes: int = 150
    num_queries: int = 100
    pixel_mean: List[float] = field(default_factory=lambda: [123.675, 116.28, 103.53])
    pixel_std: List[float] = field(default_factory=lambda: [58.395, 57.12, 57.375])
    size_divisibility: int = 0
    pixel_decoder_out_dim: int = 128
    pixel_decoder_feat_dim: int = 128
    transformer_predictor_out_dim: int = 128
    transformer_predictor_hidden_dim: int = 256
    transformer_predictor_dec_layers: int = 6
    transformer_predictor_dim_feedforward: int = 1024
    head_out_dim: int = 128
    cls_sigmoid: bool = False
    postprocessing_type: str = "semantic"
    top_k: int = 100
    mask_threshold: float = 0.5
    predict_all_pixels: bool = True
    use_mask_score: bool = False
    threshold: float = 0.5
    resolution: Optional[int] = None
    criterion_deep_supervision: bool = True
    criterion_eos_coef: float = 0.1
    criterion_num_points: int = 12544
    weight_dict_loss_dice: int = 5
    weight_dict_loss_mask: int = 5
    weight_dict_loss_ce: int = 2
    matcher_cost_class: int = 2
    matcher_cost_mask: int = 5
    matcher_cost_dice: int = 5

    @classmethod
    def from_dict(cls, d: dict) -> "BisenetFormerConfig":
        d = dict(d)
        bc = d.pop("backbone_config", {}) or {}
        if isinstance(bc, dict):
            bc = STDCConfig(**{k: v for k, v in bc.items() if k in {f.name for f in fields(STDCConfig)}})
        unknown = set(d) - {f.name for f in fields(cls)}
        if unknown:
            raise ValueError(f"Invalid parameters for BisenetFormerConfig: {sorted(unknown)}")
        return cls(backbone_config=bc, **d)


BisenetFormerOutput = MaskFormerModelOutput  # models/bisenetformer/ports.py: same fields (masks, logits, loss)


# ---- parameter containers -------------------------------------------------------------------------
class AttentionRefinementModule(nn.Module):  # bisenetformer/modelling.py:149
    def __init__(self, cin, cout):
        super().__init__()
        self.proj = nn.Conv2d(cin, cout, 1, bias=False)
        self.conv = ConvX(cout, cout, 3)
        self.conv_atten = nn.Conv2d(cout, cout, 1, bias=False)
        self.bn_atten = nn.BatchNorm2d(cout)


class ContextPath(nn.Module):  # bisenetformer/modelling.py:170
    def __init__(self, ch, d):
        super().__init__()
        self.arm32 = AttentionRefinementModule(ch[3], d)
        self.conv_avg = ConvX(ch[3], d, 1)
        self.conv_head32 = ConvX(d, d, 3)
        self.arm16 = AttentionRefinementModule(ch[2], d)
        self.conv_head16 = ConvX(d, d, 3)


class FeatureFusionModule(nn.Module):  # bisenetformer/modelling.py:213
    def __init__(self, c1, c2, cout):
        super().__init__()
        self.proj1, self.proj2 = nn.Conv2d(c1, cout, 1), nn.Conv2d(c2, cout, 1)
        self.convblk = ConvX(cout, cout, 1)
        self.conv1 = nn.Conv2d(cout, cout // 4, 1, bias=False)
        self.conv2 = nn.Conv2d(cout // 4, cout, 1, bias=False)


class BiseNet(nn.Module):  # bisenetformer/modelling.py:238
    def __init__(self, backbone: STDC, feat_dim, out_dim):
        super().__init__()
        self.backbone = backbone
        ch = backbone.out_channels
        self.cp = ContextPath(ch, feat_dim)
        self.ffm = FeatureFusionModule(ch[1], feat_dim, feat_dim)
        self.conv_out = ConvX(feat_dim, out_dim, 3)


class BisenetEngine(MFEngine):
    def _pack(self, sd):
        cfg = self.cfg
        self.nhead, self.d = 8, cfg.transformer_predictor_hidden_dim
        self.trunk = pack_trunk(self, sd)
        cp, ffm = "pixel_decoder.cp", "pixel_decoder.ffm"
        convx = lambda p: self._pack_conv(sd, p + ".conv.weight", bn=p + ".bn", act=ops.ACT_RELU)  # ConvBNReLU
        self.conv_avg = convx(cp + ".conv_avg")
        self.arm = {}
        for name in ("arm32", "arm16"):
            q = f"{cp}.{name}"
            self.arm[name] = {"proj": self._pack_conv(sd, q + ".proj.weight"), "conv": convx(q + ".conv"),
                              "att": self._pack_conv(sd, q + ".conv_atten.weight", bn=q + ".bn_atten", act=ops.ACT_SIGMOID)}
        self.head32, self.head16 = convx(cp + ".conv_head32"), convx(cp + ".conv_head16")
        self.ffm_p1 = self._pack_conv(sd, ffm + ".proj1.weight", bias=ffm + ".proj1.bias")
        self.ffm_p2 = self._pack_conv(sd, ffm + ".proj2.weight", bias=ffm + ".proj2.bias")
        self.ffm_blk = convx(ffm + ".convblk")
        self.ffm_c1 = self._pack_conv(sd, ffm + ".conv1.weight", act=ops.ACT_RELU)
        self.ffm_c2 = self._pack_conv(sd, ffm + ".conv2.weight", act=ops.ACT_SIGMOID)
        self.conv_out = convx("pixel_decoder.conv_out")
        self._pack_decoder(sd, 2)

    def _pair_layers(self):
        """the decoder linears (whether an STDC block runs in the pair format depends on its shapes: _pair_block_ok)"""
        return list(_packed_layers([self.dec, self.mask_mlp]))

    def _gate(self, conv, vec):
        """tiny [B,C] GEMM(s) of the channel-attention gates, SIMT path (M = batch size)."""
        B, C = vec.shape
        return self._conv(conv, vec.reshape(B, 1, 1, C), algo=ops.ALGO_SIMT).reshape(B, -1)

    @torch.no_grad()
    def forward(self, images: torch.Tensor, taps: Optional[dict] = None):
        B, H, W = self._input_size(images)
        # any H x W, like the reference (its processor does not resize): odd maps from the stride-2 convs and pools run on the same kernels
        _, res3, res4, res5 = self.trunk.run(images)
        res5 = _unpair(res5)  # global average pool + ARM gates work on fp32 (33 M elements at bs=64 1024x512)
        # context path; the convs that read res4 / res3 take a Pair to fp32 themselves
        avg = self._gate(self.conv_avg, ops.global_avgpool(res5))
        a = self.arm["arm32"]
        f = self._conv(a["conv"], self._conv(a["proj"], res5))
        f32 = ops.channel_scale(f, self._gate(a["att"], ops.global_avgpool(f)), addvec=avg)
        up = self._conv(self.head32, ops.resize_bilinear(f32, (res4.shape[1], res4.shape[2])))
        a = self.arm["arm16"]
        f = self._conv(a["conv"], self._conv(a["proj"], res4))
        f16 = ops.channel_scale(f, self._gate(a["att"], ops.global_avgpool(f)), addt=up)
        f8 = self._conv(self.head16, ops.resize_bilinear(f16, (res3.shape[1], res3.shape[2])))
        # feature fusion
        feat = self._conv(self.ffm_blk, self._conv(self.ffm_p1, res3, residual=self._conv(self.ffm_p2, f8)))
        att = self._gate(self.ffm_c2, self._gate(self.ffm_c1, ops.global_avgpool(feat)))
        fuse = ops.channel_scale(feat, att, self_add=True)
        mask_features = self._conv(self.conv_out, fuse)
        if taps is not None:
            taps.update(res3=_unpair(res3), res4=_unpair(res4), res5=res5, cp32=f32, cp16=f16, cp8=f8, mask_features=mask_features)
        return self._run_decoder([f32, f16], mask_features, B, H, W, taps)


class BisenetFormer(_SegmentationModel):
    """Drop-in for the reference `BisenetFormer(BaseModelNN)` (bisenetformer/modelling.py:534)."""

    engine_cls = BisenetEngine

    def __init__(self, config: BisenetFormerConfig, precision: str = "fp16"):
        c = config
        super().__init__(c, precision, BiseNet(build_trunk(c.backbone_config), c.pixel_decoder_feat_dim, c.pixel_decoder_out_dim),
                         MultiScaleMaskedTransformerDecoder(c.pixel_decoder_out_dim, c.transformer_predictor_out_dim, c.num_classes, c.transformer_predictor_hidden_dim,
                                                            c.num_queries, 8, c.transformer_predictor_dim_feedforward, c.transformer_predictor_dec_layers, 2))
