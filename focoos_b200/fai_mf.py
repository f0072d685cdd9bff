"""FAIMaskFormer (Mask2Former-style segmenter) — host-side mirror of `focoos/models/fai_mf/modelling.py` (SURVEY §8 a14-a16).

Same pattern as `fai_detr.py`: the module tree only holds parameters under the reference's state_dict keys
(SURVEY Appendix B, 937 entries for fai-mf-l-coco-ins); `FAIMaskFormer.forward` runs `MFEngine`, a fused NHWC graph:

  * ResNet-101-vd or STDC trunk (trunks.py, shared with the other families),
  * TransformerFPN pixel decoder: 1x1 input_proj -> 6 PRE-norm encoder layers with the normalised sine embedding
    (nn/layers/position_encoding.py:45-74) -> final LayerNorm -> 3x3+BN+ReLU; lateral 1x1+BN, nearest x2 upsample + add
    fused in one kernel, 3x3+BN+ReLU; mask_features 3x3 (fai_mf/modelling.py:348-369),
  * MultiScaleMaskedTransformerDecoder: 9 x (masked cross-attention -> self-attention -> FFN), pre-norm; the boolean
    attention mask is built on the device from the previous mask prediction (bilinear resize of the mask logits, `< 0`,
    all-masked rows released) and consumed by a streaming tensor-core attention kernel — the [B*8, Q, HW] bool tensor of the
    reference (:510-513) is never replicated per head,
  * PredictionHeads: LN -> class Linear / mask MLP -> per-image mask GEMM `bqc,bchw->bqhw` on tensor cores, executed
    dec_layers+1 times; intermediate class logits (dead in eval, SURVEY A.23) are skipped,
  * head: softmax[..., :-1]; sigmoid at 1/4 resolution THEN bilinear upsample to the input size, written as the reference's
    [B,Q,H,W] fp32 probability tensor by one kernel (:618-619,722-723).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, fields
from typing import List, Optional, Union

import torch
import torch.nn as nn

from . import ops
from .engine import Engine, _EngineModel, _Linear, _packed_layers, _split3_weights
from .fai_detr import MLP
from .ports import ModelOutput, ResnetConfig, STDCConfig, backbone_config_from_dict
from .trunks import STDC, ResNet, build_trunk, pack_trunk


@dataclass
class MaskFormerConfig:
    """models/fai_mf/config.py (same field names / defaults as the registry JSONs use)."""

    backbone_config: Union[ResnetConfig, STDCConfig] = field(default_factory=lambda: ResnetConfig(depth=101))
    num_classes: int = 80
    num_queries: int = 100
    resolution: Optional[int] = 1024
    pixel_mean: List[float] = field(default_factory=lambda: [123.675, 116.28, 103.53])
    pixel_std: List[float] = field(default_factory=lambda: [58.395, 57.12, 57.375])
    size_divisibility: int = 0
    pixel_decoder_out_dim: int = 256
    pixel_decoder_feat_dim: int = 256
    pixel_decoder_transformer_layers: int = 6
    pixel_decoder_transformer_dropout: float = 0.0
    pixel_decoder_transformer_nheads: int = 8
    pixel_decoder_transformer_dim_feedforward: int = 1024
    transformer_predictor_out_dim: int = 256
    transformer_predictor_hidden_dim: int = 256
    transformer_predictor_dec_layers: int = 9
    transformer_predictor_dim_feedforward: int = 2048
    head_out_dim: int = 256
    cls_sigmoid: bool = False
    postprocessing_type: str = "instance"
    mask_threshold: float = 0.5
    predict_all_pixels: bool = False
    use_mask_score: bool = True
    threshold: float = 0.5
    top_k: int = 100
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
    def from_dict(cls, d: dict) -> "MaskFormerConfig":
        d = dict(d)
        bc = backbone_config_from_dict(d.pop("backbone_config", {}), "MaskFormerConfig")
        unknown = set(d) - {f.name for f in fields(cls)}
        if unknown:
            raise ValueError(f"Invalid parameters for MaskFormerConfig: {sorted(unknown)}")
        return cls(backbone_config=bc, **d)


@dataclass
class MaskFormerModelOutput(ModelOutput):
    """models/fai_mf/ports.py: field order (masks, logits, loss)."""

    masks: torch.Tensor  # [B, Q, H, W] fp32 probabilities at the input resolution
    logits: torch.Tensor  # [B, Q, num_classes] softmax probabilities without the no-object column
    loss: Optional[dict] = None


class LazyMasks:
    """The model output `masks` before the final sigmoid + bilinear upsampling (fai_mf/modelling.py:619,722-723): low-resolution logits
    NHWC [B,h,w,Qp] plus the target size.  `materialize()` gives the reference's [B,Q,H,W] fp32 probabilities; a processor that understands
    this object fuses the upsampling into its own reduction instead (semantic argmax: 13.4 GB of HBM traffic avoided at config 4).
    Enabled by `model.lazy_masks = True` (FocoosModel sets it: it owns model + processor); plain `model(images)` returns tensors."""

    def __init__(self, logits_nhwc: torch.Tensor, num_queries: int, size):
        self.logits, self.num_queries, self.size = logits_nhwc, num_queries, (int(size[0]), int(size[1]))

    @property
    def shape(self):
        return (self.logits.shape[0], self.num_queries, *self.size)

    @property
    def device(self):
        return self.logits.device

    def materialize(self) -> torch.Tensor:
        return ops.mask_sigmoid_upsample(self.logits, self.num_queries, self.size)


# ---- parameter containers -------------------------------------------------------------------------
class _ConvBN(nn.Conv2d):
    """nn/layers/conv.py:22 `Conv2d` wrapper whose norm is a CHILD module (`<name>.weight`, `<name>.norm.*`)."""

    def __init__(self, cin, cout, k, bias=False, norm=True):
        super().__init__(cin, cout, k, padding=(k - 1) // 2, bias=bias)
        self.norm = nn.BatchNorm2d(cout) if norm else None


class _EncLayer(nn.Module):
    def __init__(self, d, nhead, dff):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d, nhead, 0.0)
        self.linear1, self.linear2 = nn.Linear(d, dff), nn.Linear(dff, d)
        self.norm1, self.norm2 = nn.LayerNorm(d), nn.LayerNorm(d)


class _Encoder(nn.Module):
    def __init__(self, d, nhead, dff, n):
        super().__init__()
        self.layers = nn.ModuleList([_EncLayer(d, nhead, dff) for _ in range(n)])
        self.norm = nn.LayerNorm(d)


class _EncoderOnly(nn.Module):  # fai_mf/modelling.py:130
    def __init__(self, d, nhead, dff, n):
        super().__init__()
        self.encoder = _Encoder(d, nhead, dff, n)


class TransformerFPN(nn.Module):  # fai_mf/modelling.py:201
    def __init__(self, backbone: Union[ResNet, STDC], feat_dim, out_dim, layers, nhead, dff):
        super().__init__()
        self.backbone = backbone
        ch = backbone.out_channels  # res2..res5
        if layers > 0:
            self.input_proj = _ConvBN(ch[3], feat_dim, 1, bias=True, norm=False)
            self.transformer = _EncoderOnly(feat_dim, nhead, dff, layers)
        for idx in (1, 2, 3):
            self.add_module(f"adapter_{idx}", _ConvBN(ch[idx - 1], feat_dim, 1))
            self.add_module(f"layer_{idx}", _ConvBN(feat_dim, feat_dim, 3))
        # without an encoder (fai-mf-*-ade: :241-284) layer_4 reads res5 itself
        self.layer_4 = _ConvBN(feat_dim if layers > 0 else ch[3], feat_dim, 3)
        self.mask_features = _ConvBN(feat_dim, out_dim, 3, bias=True, norm=False)


class _AttnLayer(nn.Module):
    def __init__(self, d, nhead, name):
        super().__init__()
        setattr(self, name, nn.MultiheadAttention(d, nhead, dropout=0.0))
        self.norm = nn.LayerNorm(d)


class _FFNLayer(nn.Module):
    def __init__(self, d, dff):
        super().__init__()
        self.linear1, self.linear2, self.norm = nn.Linear(d, dff), nn.Linear(dff, d), nn.LayerNorm(d)


class PredictionHeads(nn.Module):  # fai_mf/modelling.py:28
    def __init__(self, d, num_classes, mask_dim):
        super().__init__()
        self.decoder_norm = nn.LayerNorm(d)
        self.classifier = nn.Linear(d, num_classes + 1)
        self.mask_classifier = MLP(d, d, mask_dim, 3)


class MultiScaleMaskedTransformerDecoder(nn.Module):  # fai_mf/modelling.py:372; bisenetformer/modelling.py:285 (TransformerDecoder, two levels)
    def __init__(self, in_ch, out_dim, num_classes, d, num_queries, nhead, dff, layers, levels=3):
        super().__init__()
        self.transformer_self_attention_layers = nn.ModuleList([_AttnLayer(d, nhead, "self_attn") for _ in range(layers)])
        self.transformer_cross_attention_layers = nn.ModuleList([_AttnLayer(d, nhead, "multihead_attn") for _ in range(layers)])
        self.transformer_ffn_layers = nn.ModuleList([_FFNLayer(d, dff) for _ in range(layers)])
        self.query_feat, self.query_embed = nn.Embedding(num_queries, d), nn.Embedding(num_queries, d)
        self.input_proj = nn.ModuleList([_ConvBN(in_ch, d, 1, bias=True, norm=False) for _ in range(levels)])
        self.forward_prediction_heads = PredictionHeads(d, num_classes, out_dim)


def position_embedding_sine_normalized(h, w, num_pos_feats=128, temperature=10000.0):
    """nn/layers/position_encoding.py:45-74, normalize=True -> [h*w, 2*num_pos_feats] (token-major for the NHWC graph)."""
    y = torch.arange(1, h + 1, dtype=torch.float32).view(h, 1).expand(h, w)
    x = torch.arange(1, w + 1, dtype=torch.float32).view(1, w).expand(h, w)
    eps, scale = 1e-6, 2 * math.pi
    y = y / (float(h) + eps) * scale
    x = x / (float(w) + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    px, py = x[:, :, None] / dim_t, y[:, :, None] / dim_t
    px = torch.stack((px[:, :, 0::2].sin(), px[:, :, 1::2].cos()), dim=3).view(h, w, -1)
    py = torch.stack((py[:, :, 0::2].sin(), py[:, :, 1::2].cos()), dim=3).view(h, w, -1)
    return torch.cat((py, px), dim=2).reshape(h * w, -1)


class MFEngine(Engine):
    """Packs a FAIMaskFormer state_dict and runs the fused forward: trunk, TransformerFPN pixel decoder, masked transformer decoder and head."""

    lazy_masks = False  # True: return LazyMasks instead of the materialised [B,Q,H,W] probabilities

    def _pack(self, sd):
        cfg = self.cfg
        self.nhead, self.d = 8, cfg.transformer_predictor_hidden_dim  # masked decoder
        # the pixel-decoder encoder has its own width and heads: 256 x 8 heads of 32 channels (fai-mf-l), 128 x 8 heads of 16 channels (fai-mf-m / -s)
        self.pd_d, self.pd_nhead = cfg.pixel_decoder_feat_dim, cfg.pixel_decoder_transformer_nheads
        self.trunk = pack_trunk(self, sd)
        pd = "pixel_decoder"
        # no encoder (fai-mf-*-ade): no input_proj, no encoder layers, no final LayerNorm - layer_4 reads res5
        self.pd_in = self.enc_norm = None
        self.enc = [self._pack_attn_block(sd, f"{pd}.transformer.encoder.layers.{i}", ffn_norms=("norm1", "norm2"), d=self.pd_d)
                    for i in range(cfg.pixel_decoder_transformer_layers)]
        if self.enc:
            self.pd_in = self._pack_conv(sd, pd + ".input_proj.weight", bias=pd + ".input_proj.bias")
            self.enc_norm = (self._f32(sd[pd + ".transformer.encoder.norm.weight"]), self._f32(sd[pd + ".transformer.encoder.norm.bias"]))
        self.layer = {i: self._pack_conv(sd, f"{pd}.layer_{i}.weight", bn=f"{pd}.layer_{i}.norm", act=ops.ACT_RELU) for i in (1, 2, 3, 4)}
        self.adapter = {i: self._pack_conv(sd, f"{pd}.adapter_{i}.weight", bn=f"{pd}.adapter_{i}.norm") for i in (1, 2, 3)}
        self.mask_features = self._pack_conv(sd, pd + ".mask_features.weight", bias=pd + ".mask_features.bias")
        self._pack_decoder(sd, 3)

    def _pair_layers(self):
        """the trunk's pair layers (on an STDC trunk, whether a block runs on pairs is _pair_block_ok's call), the pixel-decoder convs that read its
        pairs, the 1/4-resolution chain into mask_features, and the decoder linears.  res5 is read by input_proj, or without an encoder by layer_4 itself."""
        res5_reader = self.pd_in if self.enc else self.layer[4]
        return self.trunk.pair_layers() + list(_packed_layers([res5_reader, self.adapter, self.layer[1], self.mask_features, self.dec, self.mask_mlp]))

    def _pack_decoder(self, sd, num_levels):
        """head.predictor.* of the masked transformer decoder (same key names in fai_mf and bisenetformer)."""
        cfg = self.cfg
        hp = "head.predictor"
        self.dec_in = [self._pack_conv(sd, f"{hp}.input_proj.{i}.weight", bias=f"{hp}.input_proj.{i}.bias") for i in range(num_levels)]
        self.query_feat, self.query_embed = self._to(sd[hp + ".query_feat.weight"].float()), self._to(sd[hp + ".query_embed.weight"].float())
        d = self.d
        self.dec = []
        for i in range(cfg.transformer_predictor_dec_layers):
            c, s, f = (f"{hp}.transformer_cross_attention_layers.{i}", f"{hp}.transformer_self_attention_layers.{i}", f"{hp}.transformer_ffn_layers.{i}")
            wc, bc = sd[c + ".multihead_attn.in_proj_weight"].float(), sd[c + ".multihead_attn.in_proj_bias"].float()
            ws, bs = sd[s + ".self_attn.in_proj_weight"].float(), sd[s + ".self_attn.in_proj_bias"].float()
            self.dec.append({
                "cq": _Linear(self._to(wc[:d]), self._f32(bc[:d])), "ck": _Linear(self._to(wc[d:2 * d]), self._f32(bc[d:2 * d])),
                "cv": _Linear(self._to(wc[2 * d:]), self._f32(bc[2 * d:])), "cout": self._lin(sd, c + ".multihead_attn.out_proj"),
                "cn": (self._f32(sd[c + ".norm.weight"]), self._f32(sd[c + ".norm.bias"])),
                "sqk": _Linear(self._to(ws[:2 * d]), self._f32(bs[:2 * d])), "sv": _Linear(self._to(ws[2 * d:]), self._f32(bs[2 * d:])),
                "sout": self._lin(sd, s + ".self_attn.out_proj"), "sn": (self._f32(sd[s + ".norm.weight"]), self._f32(sd[s + ".norm.bias"])),
                "l1": self._lin(sd, f + ".linear1"), "l2": self._lin(sd, f + ".linear2"), "fn": (self._f32(sd[f + ".norm.weight"]), self._f32(sd[f + ".norm.bias"])),
            })
        h = hp + ".forward_prediction_heads"
        self.head_norm = (self._f32(sd[h + ".decoder_norm.weight"]), self._f32(sd[h + ".decoder_norm.bias"]))
        self.classifier = self._lin(sd, h + ".classifier")
        self.mask_mlp = [self._lin(sd, f"{h}.mask_classifier.layers.{j}") for j in range(3)]

    def _pos(self, h, w, d=None):
        """the normalised sine embedding of an h x w map for a d-wide sequence (default: the decoder width self.d)"""
        d = self.d if d is None else d
        key = ("pos", h, w, d)
        if key not in self._consts:
            self._consts[key] = self._to(position_embedding_sine_normalized(h, w, d // 2))
        return self._consts[key]

    def _heads(self, out, mask_features, size, want_class):
        """PredictionHeads.forward (:69-112) -> (class logits fp32 or None, mask logits NHWC [B,h4,w4,Qp], (mask, allowed) or None).
        mask_features: a Pair under fp32_tc (see _run_decoder)."""
        A, dt = self.algo, self.dt
        B, Q, d = out.shape
        dn, dnp, _ = self._norm(out, self.head_norm, want_f32=want_class)
        cls = self._linear(self.classifier, dn, out_dtype=torch.float32, algo=ops.ALGO_SIMT) if want_class else None
        me = self._mlp(self.mask_mlp, dnp)  # [B,Q,256]
        _, h4, w4, C = mask_features.shape
        Qp = (Q + 7) // 8 * 8
        masks = torch.zeros((B, h4, w4, Qp), dtype=dt, device=out.device)
        # einsum("bqc,bchw->bqhw"): a [h4*w4, C] x [C, Q] GEMM per image whose "weights" (the mask embeddings) differ per image - ONE launch
        if self.pair:
            # the same GEMM as three fp16 tensor-core products on the mask_features pair and the per-image embeddings as [W_hi | W_lo | W_hi] triples.
            # (On the CUDA-core fp32 kernel this product was a third of the parity-mode step: 16.9 of 50.4 ms at bs=16 800x800.)
            ops.conv2d_per_image(mask_features, _split3_weights(me).reshape(B, Q, 1, 1, 3 * C), out=masks[..., :Q])
        elif dt == torch.float16 and Qp != Q:
            # the fp16 tensor-core store writes whole 16-byte pieces (8 channels): the product runs on all Qp columns, zero embeddings past Q, so that
            # it owns every column it writes
            ops.conv2d_per_image(mask_features, nn.functional.pad(me, (0, 0, 0, Qp - Q)).reshape(B, Qp, 1, 1, C), out=masks, algo=A)
        else:
            ops.conv2d_per_image(mask_features, me.reshape(B, Q, 1, 1, C), out=masks[..., :Q], algo=A)
        attn = None
        if size is not None:
            low = masks if (h4, w4) == tuple(size) else ops.resize_bilinear(masks, size)
            attn = ops.attn_mask_build(low, Q)
        return cls, masks, attn

    @torch.no_grad()
    def forward(self, images: torch.Tensor, taps: Optional[dict] = None):
        B, H, W = self._input_size(images)
        # any H x W, like the reference (its processor does not resize): odd maps from the stride-2 convs and ceil-mode pools run on the same kernels
        # fp32_tc: the backbone keeps its activations as fp16 [hi | lo] planes between convs (no split pass in front of every conv); the four pixel-decoder
        # convs that consume res2..res5 read the pairs and write the fp32 tensors the transformer / FPN arithmetic below works on
        res2, res3, res4, res5 = self.trunk.run(images)
        d, nh = self.pd_d, self.pd_nhead
        scale = 1.0 / math.sqrt(d // nh)
        # ---- pixel decoder (TransformerFPN.forward_features)
        if self.enc:
            x = self._conv(self.pd_in, res5)
            h, w = x.shape[1], x.shape[2]
            pos = self._pos(h, w, d)
            src = x.reshape(B, h * w, d)
            for blk in self.enc:  # pre-norm encoder layer (nn/layers/transformer.py:583-601 with normalize_before)
                s2 = ops.layernorm(src, *blk["n_attn"])
                qk = self._linear(blk["qk"], ops.add(s2, pos))
                a = ops.attention(qk[..., :d], qk[..., d:], self._linear(blk["v"], s2), nh, scale, split=self.pair)
                src = self._linear(blk["out"], a, residual=src)
                s2 = ops.layernorm(src, *blk["n_ffn"])
                src = self._linear(blk["l2"], self._linear(blk["l1"], s2, act=ops.ACT_RELU), residual=src)
            src = ops.layernorm(src, *self.enc_norm)
            y = self._conv(self.layer[4], src.reshape(B, h, w, d))
        else:  # no encoder: the 3x3 output conv reads res5 (a Pair under fp32_tc)
            y = self._conv(self.layer[4], res5)
        ms = [y]
        # fp32_tc: the 1/4-resolution layer feeds only the mask_features conv, whose output is only ever read as a tensor-core operand (the per-image mask product):
        # both stay in the pair format - no fp32 copy of the two largest activations of the pixel decoder, no split pass over them
        for idx, f in ((3, res4), (2, res3), (1, res2)):
            u = ops.upsample_nearest_add(y, self._conv(self.adapter[idx], f))
            y = self._conv(self.layer[idx], u, out_pair=idx == 1)
            if len(ms) < 3:
                ms.append(y)
        mask_features = self._conv(self.mask_features, y, out_pair=True)
        if taps is not None:
            taps.update(res5=res5.float(), mask_features=mask_features.float(), multi_scale=ms)
            if self.enc:
                taps["enc_memory"] = src.reshape(B, h, w, d)
        return self._run_decoder(ms, mask_features, B, H, W, taps)

    def _run_decoder(self, ms, mask_features, B, H, W, taps=None):
        """MultiScaleMaskedTransformerDecoder.forward (fai_mf/modelling.py:467-550) + head + final upsample; `ms` = the decoder's
        feature levels (3 for fai_mf, 2 for bisenetformer)."""
        cfg = self.cfg
        d, nh = self.d, self.nhead
        scale = 1.0 / math.sqrt(d // nh)
        nl = len(ms)
        if self.pair:  # every _heads call reads mask_features as a Pair: MaskFormer's conv writes one, BisenetFormer's fp32 output is split once here
            # the tensor-core product takes channel counts in 32-channel chunks (bisenetformer-m-ade: 96 = 3 chunks per plane)
            assert mask_features.shape[-1] % 32 == 0, mask_features.shape
            mask_features = ops.to_pair(mask_features)
        srcs, kpos, sizes = [], [], []
        for i in range(nl):
            hh, ww = ms[i].shape[1], ms[i].shape[2]
            s = self._conv(self.dec_in[i], ms[i]).reshape(B, hh * ww, d)
            srcs.append(s)
            kpos.append(ops.add(s, self._pos(hh, ww)))
            sizes.append((hh, ww))
        Q = cfg.num_queries
        out = self.query_feat.unsqueeze(0).expand(B, Q, d).contiguous()
        qpos = self.query_embed
        L = len(self.dec)
        cls = None
        # fp32_tc: the per-level key / value inputs are split once (every layer of a level reads the same ones), the K / V projections run pair -> pair
        kpos, srcs = [self._operand(t) for t in kpos], [self._operand(t) for t in srcs]
        _, masks, attn = self._heads(out, mask_features, sizes[0], False)
        for i, blk in enumerate(self.dec):
            lvl = i % nl
            _, _, tq = self._norm(out, blk["cn"], pos=qpos, want_f32=False, want_op=False)
            q = self._linear(blk["cq"], tq)
            kk, vv = self._linear(blk["ck"], kpos[lvl], out_pair=True), self._linear(blk["cv"], srcs[lvl], out_pair=True)
            a = ops.attention_masked(q, kk, vv, attn[0], attn[1], nh, scale, split=self.pair)
            out = self._linear(blk["cout"], self._operand(a), residual=out)
            _, t2, t2p = self._norm(out, blk["sn"], pos=qpos, want_f32=False)
            qk = self._linear(blk["sqk"], t2p)
            a = ops.attention(qk[..., :d], qk[..., d:], self._linear(blk["sv"], t2), nh, scale, split=self.pair, out_pair=self.pair)
            out = self._linear(blk["sout"], a, residual=out)
            _, ffn_in, _ = self._norm(out, blk["fn"], want_f32=False)
            out = self._linear(blk["l2"], self._linear(blk["l1"], ffn_in, act=ops.ACT_RELU, out_pair=True), residual=out)
            last = i == L - 1
            cls, masks, attn = self._heads(out, mask_features, None if last else sizes[(i + 1) % nl], last)
            if taps is not None:
                taps[f"dec{i}_out"] = out
        if taps is not None:
            taps.update(pred_logits=cls, pred_masks=masks)  # masks: NHWC [B,h4,w4,Qp] pre-sigmoid logits
        probs = ops.softmax_drop_last(cls)
        lazy = LazyMasks(masks, Q, (H, W))
        return probs, (lazy if self.lazy_masks else lazy.materialize())


class _SegmentationModel(_EngineModel):
    """What FAIMaskFormer and BisenetFormer share: inference through the engine, masks returned as LazyMasks when `lazy_masks` is set."""

    lazy_masks = False  # True: forward() returns fai_mf.LazyMasks (low-resolution logits) instead of the upsampled [B,Q,H,W] probabilities

    def forward(self, images: torch.Tensor, targets: list = [], taps: Optional[dict] = None) -> MaskFormerModelOutput:
        if self.training or (targets is not None and len(targets) > 0):
            raise NotImplementedError("focoos_b200: losses / fine-tuning are not part of the inference hot path")
        self._check_device(images)
        eng = self.engine()
        eng.lazy_masks = bool(getattr(self, "lazy_masks", False))
        probs, masks = eng.forward(images if images.dtype == torch.uint8 else images.to(torch.float32), taps)
        return MaskFormerModelOutput(masks=masks, logits=probs, loss=None)


class FAIMaskFormer(_SegmentationModel):
    """Drop-in for the reference `FAIMaskFormer(BaseModelNN)` (fai_mf/modelling.py:633)."""

    engine_cls = MFEngine

    def __init__(self, config: MaskFormerConfig, precision: str = "fp16"):
        c = config
        if c.postprocessing_type not in ("semantic", "instance"):
            raise ValueError(f"Invalid postprocessing type: {c.postprocessing_type}. Must be one of: ['semantic', 'instance']")
        super().__init__(c, precision,
                         TransformerFPN(build_trunk(c.backbone_config), c.pixel_decoder_feat_dim, c.pixel_decoder_out_dim, c.pixel_decoder_transformer_layers,
                                        c.pixel_decoder_transformer_nheads, c.pixel_decoder_transformer_dim_feedforward),
                         MultiScaleMaskedTransformerDecoder(c.pixel_decoder_out_dim, c.transformer_predictor_out_dim, c.num_classes, c.transformer_predictor_hidden_dim,
                                                            c.num_queries, 8, c.transformer_predictor_dim_feedforward, c.transformer_predictor_dec_layers))
