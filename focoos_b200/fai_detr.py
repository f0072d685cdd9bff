"""FAIDetr (RT-DETR-style detector) — host-side mirror of `focoos/models/fai_detr/modelling.py`.

The module TREE below mirrors the reference's (same attribute names, same parameter shapes) so that a
reference `state_dict` / `model_final.pth` loads unchanged (SURVEY.md Appendix B), but the modules are only
parameter containers: `FAIDetr.forward` runs `DetrEngine`, a fused NHWC graph of `focoos_b200.ops`
calls (hand-written sm_90a kernels) built once from the weights:

  * BatchNorm folded into per-channel scale/bias applied in the conv epilogue (nn/layers/conv.py:89),
  * RepVggBlock re-parameterised to one 3x3 conv (the reference's own `get_equivalent_kernel_bias`,
    modelling.py:57-61, which it never calls),
  * CSPRepLayer conv1‖conv2 as ONE 1x1 GEMM (N=512) and its output add fused as a post-activation residual,
  * concat-free FPN/PAN: producers write straight into channel slices of the concat buffer,
  * the six decoder value_proj GEMMs batched into one (memory is layer-invariant, modelling.py:848),
  * sampling_offsets ‖ attention_weights as one GEMM feeding the fused MSDA kernel,
  * encoder bbox MLP evaluated only on the 300 selected rows (row-wise op; identical result),
  * the dead `mask_features` conv (modelling.py:347 computed, :381 discarded) skipped.

There is no CPU / eager fallback: `forward` raises unless the tensors are on a CUDA device and the
compiled library is present.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .engine import Engine, _bn_fold, _channels, _Conv, _EngineModel, _Linear, _pad_rows, _packed_layers, _unpair
from .ports import DETRConfig, DETRModelOutput
from .trunks import ConvNormLayer, build_trunk, pack_trunk
# these lived here before engine.py / trunks.py existed; bench.py and code written against that layout import them from this module
from .engine import _split3_weights  # noqa: F401,E402
from .trunks import STDC, ResNet  # noqa: F401,E402

NUM_POINTS = 4  # num_decoder_points (modelling.py:1039): sampling points per head and level of the deformable cross-attention


# --------------------------------------------------------------------------------------------------
# parameter containers (names = the reference's state_dict keys)
# --------------------------------------------------------------------------------------------------
class RepVggBlock(nn.Module):  # modelling.py:30
    def __init__(self, ch):
        super().__init__()
        self.conv1 = ConvNormLayer(ch, ch, 3, 1)
        self.conv2 = ConvNormLayer(ch, ch, 1, 1)


class CSPRepLayer(nn.Module):  # modelling.py:84 (expansion 1.0 -> conv3 = Identity)
    def __init__(self, ch_in, ch_out, num_blocks=3):
        super().__init__()
        self.conv1 = ConvNormLayer(ch_in, ch_out, 1, 1, "silu")
        self.conv2 = ConvNormLayer(ch_in, ch_out, 1, 1, "silu")
        self.bottlenecks = nn.Sequential(*[RepVggBlock(ch_out) for _ in range(num_blocks)])
        self.conv3 = nn.Identity()


class TransformerEncoderLayer(nn.Module):  # nn/layers/transformer.py:553
    def __init__(self, d, nhead, dff):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d, nhead, 0.0, batch_first=True)
        self.linear1, self.linear2 = nn.Linear(d, dff), nn.Linear(dff, d)
        self.norm1, self.norm2 = nn.LayerNorm(d), nn.LayerNorm(d)


class TransformerEncoder(nn.Module):  # nn/layers/transformer.py:471
    def __init__(self, d, nhead, dff, n):
        super().__init__()
        self.layers = nn.ModuleList([TransformerEncoderLayer(d, nhead, dff) for _ in range(n)])


class Encoder(nn.Module):  # modelling.py:195 ("pixel_decoder")
    def __init__(self, backbone, feat_dim, out_dim, nhead, dff, num_encoder_layers):
        """backbone: ResNet or STDC; the input projections read its res3 / res4 / res5 channels.  num_encoder_layers 0 holds no AIFI parameters."""
        super().__init__()
        self.backbone = backbone
        in_ch = backbone.out_channels[1:]
        self.input_proj = nn.ModuleList([nn.Sequential(nn.Conv2d(c, feat_dim, 1, bias=False), nn.BatchNorm2d(feat_dim)) for c in in_ch])
        self.encoder = nn.ModuleList([TransformerEncoder(feat_dim, nhead, dff, num_encoder_layers)])
        self.lateral_convs = nn.ModuleList([ConvNormLayer(feat_dim, feat_dim, 1, 1, "silu") for _ in range(2)])
        self.fpn_blocks = nn.ModuleList([CSPRepLayer(feat_dim * 2, feat_dim) for _ in range(2)])
        self.downsample_convs = nn.ModuleList([ConvNormLayer(feat_dim, feat_dim, 3, 1, "silu") for _ in range(2)])
        self.pan_blocks = nn.ModuleList([CSPRepLayer(feat_dim * 2, feat_dim) for _ in range(2)])
        self.mask_features = nn.Conv2d(feat_dim, out_dim, 3, 1, 1)  # dead for detection (modelling.py:381); kept for the weight file


class MLP(nn.Module):  # nn/layers/base.py:31
    def __init__(self, i, h, o, n):
        super().__init__()
        hs = [h] * (n - 1)
        self.layers = nn.ModuleList(nn.Linear(a, b) for a, b in zip([i] + hs, hs + [o]))


class MSDeformableAttention(nn.Module):  # modelling.py:777
    def __init__(self, d, heads, levels, points):
        super().__init__()
        self.sampling_offsets = nn.Linear(d, heads * levels * points * 2)
        self.attention_weights = nn.Linear(d, heads * levels * points)
        self.value_proj, self.output_proj = nn.Linear(d, d), nn.Linear(d, d)


class TransformerDecoderLayer(nn.Module):  # modelling.py:887
    def __init__(self, d, heads, dff, levels, points):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d, heads, dropout=0.0, batch_first=True)
        self.norm1 = nn.LayerNorm(d)
        self.cross_attn = MSDeformableAttention(d, heads, levels, points)
        self.norm2 = nn.LayerNorm(d)
        self.linear1, self.linear2 = nn.Linear(d, dff), nn.Linear(dff, d)
        self.norm3 = nn.LayerNorm(d)


class TransformerDecoder(nn.Module):  # modelling.py:961
    def __init__(self, d, heads, dff, levels, points, n):
        super().__init__()
        self.layers = nn.ModuleList([TransformerDecoderLayer(d, heads, dff, levels, points) for _ in range(n)])


class TransformerPredictor(nn.Module):  # modelling.py:1023
    def __init__(self, in_channels, num_classes, hidden, num_queries, nhead, dec_layers, dff, num_scales=3, points=4):
        super().__init__()
        self.num_queries, self.num_levels, self.num_points, self.nhead, self.dec_layers = num_queries, num_scales, points, nhead, dec_layers
        self.input_proj = nn.ModuleList([
            nn.Sequential(OrderedDict([("conv", nn.Conv2d(in_channels, hidden, 1, bias=False)), ("norm", nn.BatchNorm2d(hidden))]))
            for _ in range(num_scales)])
        self.decoder = TransformerDecoder(hidden, nhead, dff, num_scales, points, dec_layers)
        self.query_pos_head = MLP(4, 2 * hidden, hidden, 2)
        self.enc_output = nn.Sequential(nn.Linear(hidden, hidden), nn.LayerNorm(hidden))
        self.enc_score_classifier = nn.Linear(hidden, num_classes)
        self.enc_bbox_classifier = MLP(hidden, hidden, 4, 3)
        self.dec_score_classifier = nn.ModuleList([nn.Linear(hidden, num_classes) for _ in range(dec_layers)])
        self.dec_bbox_classifier = nn.ModuleList([MLP(hidden, hidden, 4, 3) for _ in range(dec_layers)])


def generate_anchors(spatial_shapes, grid_size=0.05, eps=1e-2):
    """modelling.py:1169-1189 — logit-space anchors [S,4] fp32 and validity [S] (host, once per resolution)."""
    anchors = []
    for lvl, (h, w) in enumerate(spatial_shapes):
        gy, gx = torch.meshgrid(torch.arange(end=h, dtype=torch.float32), torch.arange(end=w, dtype=torch.float32), indexing="ij")
        grid_xy = (torch.stack([gx, gy], -1).unsqueeze(0) + 0.5) / torch.tensor([w, h], dtype=torch.float32)
        wh = torch.ones_like(grid_xy) * grid_size * (2.0 ** (2 - lvl))
        anchors.append(torch.concat([grid_xy, wh], -1).reshape(-1, h * w, 4))
    anchors = torch.concat(anchors, 1)
    valid = ((anchors > eps) * (anchors < 1 - eps)).all(-1, keepdim=True)
    anchors = torch.where(valid, torch.log(anchors / (1 - anchors)), torch.zeros(()))
    return anchors[0].contiguous(), valid[0, :, 0].contiguous()


def aifi_position_embedding(h, w, num_pos_feats=128, temperature=10000.0):
    """modelling.py:110-179 with normalize=False: [h*w, 4*num_pos_feats/2] = cat(y_sin, y_cos, x_sin, x_cos)."""
    y_embed = torch.arange(h, dtype=torch.float32).view(h, 1).expand(h, w)
    x_embed = torch.arange(w, dtype=torch.float32).view(1, w).expand(h, w)
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    pos_x = x_embed[:, :, None] / dim_t
    pos_y = y_embed[:, :, None] / dim_t
    return torch.cat((pos_y[:, :, 0::2].sin().reshape(h * w, -1), pos_y[:, :, 1::2].cos().reshape(h * w, -1),
                      pos_x[:, :, 0::2].sin().reshape(h * w, -1), pos_x[:, :, 1::2].cos().reshape(h * w, -1)), dim=1)


# --------------------------------------------------------------------------------------------------
# the fused graph
# --------------------------------------------------------------------------------------------------
class DetrEngine(Engine):
    """Packs a FAIDetr state_dict and runs the fused forward: trunk, hybrid encoder, query selection, deformable decoder and head."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if self.pair:
            # the pair flow's score head (_forward_head) writes the class logits into rows padded to 16 bytes (the tensor-core store writes whole
            # 16-byte pieces): zero rows up to that width make the launch own every column it stores
            self.dec_score = _pad_rows(self.dec_score, 4)

    def _pair_layers(self):
        """the packed layers the fp32_tc flow runs on their weight triples: all but the trunk's stem (stem_conv) and query_pos_head.layers.0 (K = 4),
        which stay fp32"""
        return [layer for layer in _packed_layers(vars(self)) if layer is not self.qpos[0] and layer is not self.trunk.stem]

    def _csp(self, sd, p):
        w1, w2 = sd[p + ".conv1.conv.weight"].float(), sd[p + ".conv2.conv.weight"].float()
        s1, b1 = _bn_fold(sd, p + ".conv1.norm")
        s2, b2 = _bn_fold(sd, p + ".conv2.norm")
        both = _Conv(self._to(torch.cat([w1, w2], 0).permute(0, 2, 3, 1)), self._f32(torch.cat([s1, s2])), self._f32(torch.cat([b1, b2])), 1, 0, ops.ACT_SILU)
        reps = []
        i = 0
        while f"{p}.bottlenecks.{i}.conv1.conv.weight" in sd:
            q = f"{p}.bottlenecks.{i}"
            s3, b3 = _bn_fold(sd, q + ".conv1.norm")
            s1_, b1_ = _bn_fold(sd, q + ".conv2.norm")
            k = sd[q + ".conv1.conv.weight"].float() * s3.view(-1, 1, 1, 1) + nn.functional.pad(sd[q + ".conv2.conv.weight"].float() * s1_.view(-1, 1, 1, 1), [1, 1, 1, 1])
            reps.append(_Conv(self._to(k.permute(0, 2, 3, 1)), None, self._f32(b3 + b1_), 1, 1, ops.ACT_SILU))
            i += 1
        return both, reps

    def _pack(self, sd):
        cfg = self.cfg
        self.nhead, self.d = cfg.transformer_predictor_nhead, cfg.transformer_predictor_hidden_dim
        self.trunk = pack_trunk(self, sd)
        pd = "pixel_decoder"
        self.enc_in = [self._pack_conv(sd, f"{pd}.input_proj.{i}.0.weight", bn=f"{pd}.input_proj.{i}.1") for i in range(3)]
        # the AIFI layer on the 1/32 map (fai-detr-l-*); fai-detr-m-coco has none (pixel_decoder_num_encoder_layers 0)
        self.aifi = self._pack_attn_block(sd, f"{pd}.encoder.0.layers.0", ffn_norms=("norm1", "norm2")) if cfg.pixel_decoder_num_encoder_layers else None
        self.lateral = [self._pack_conv(sd, f"{pd}.lateral_convs.{i}.conv.weight", bn=f"{pd}.lateral_convs.{i}.norm", act=ops.ACT_SILU) for i in range(2)]
        self.fpn = [self._csp(sd, f"{pd}.fpn_blocks.{i}") for i in range(2)]
        self.down = [self._pack_conv(sd, f"{pd}.downsample_convs.{i}.conv.weight", bn=f"{pd}.downsample_convs.{i}.norm", act=ops.ACT_SILU) for i in range(2)]
        self.pan = [self._csp(sd, f"{pd}.pan_blocks.{i}") for i in range(2)]
        hp = "head.predictor"
        self.dec_in = [self._pack_conv(sd, f"{hp}.input_proj.{i}.conv.weight", bn=f"{hp}.input_proj.{i}.norm") for i in range(3)]
        self.enc_output = self._lin(sd, hp + ".enc_output.0")
        self.enc_output_ln = (self._f32(sd[hp + ".enc_output.1.weight"]), self._f32(sd[hp + ".enc_output.1.bias"]))
        self.enc_score = self._lin(sd, hp + ".enc_score_classifier")
        self.enc_bbox = [self._lin(sd, f"{hp}.enc_bbox_classifier.layers.{i}") for i in range(3)]
        self.qpos = [self._lin(sd, hp + ".query_pos_head.layers.0", dtype=torch.float32), self._lin(sd, hp + ".query_pos_head.layers.1")]
        L = self.cfg.transformer_predictor_dec_layers
        vw = torch.cat([sd[f"{hp}.decoder.layers.{i}.cross_attn.value_proj.weight"].float() for i in range(L)], 0)
        vb = torch.cat([sd[f"{hp}.decoder.layers.{i}.cross_attn.value_proj.bias"].float() for i in range(L)], 0)
        self.value_all = _Linear(self._to(vw), self._f32(vb))
        self.dec = []
        for i in range(L):
            p = f"{hp}.decoder.layers.{i}"
            blk = self._pack_attn_block(sd, p, ffn_norms=("norm1", "norm3"))
            oa_w = torch.cat([sd[p + ".cross_attn.sampling_offsets.weight"].float(), sd[p + ".cross_attn.attention_weights.weight"].float()], 0)
            oa_b = torch.cat([sd[p + ".cross_attn.sampling_offsets.bias"].float(), sd[p + ".cross_attn.attention_weights.bias"].float()], 0)
            blk["oa"] = _Linear(self._to(oa_w), self._f32(oa_b))
            blk["cross_out"] = self._lin(sd, p + ".cross_attn.output_proj")
            blk["n_cross"] = (self._f32(sd[p + ".norm2.weight"]), self._f32(sd[p + ".norm2.bias"]))
            blk["bbox"] = [self._lin(sd, f"{hp}.dec_bbox_classifier.{i}.layers.{j}") for j in range(3)]
            self.dec.append(blk)
        self.dec_score = self._lin(sd, f"{hp}.dec_score_classifier.{L - 1}")

    def _constants(self, h32, w32):
        key = (h32, w32)
        if key not in self._consts:
            shapes = [(h32, w32), (h32 * 2, w32 * 2), (h32 * 4, w32 * 4)]
            anchors, valid = generate_anchors(shapes)
            self._consts[key] = {"shapes": shapes, "anchors": self._f32(anchors), "valid": valid.to(self.device, torch.uint8).contiguous()}
            if self.aifi is not None:
                self._consts[key]["pos"] = self._to(aifi_position_embedding(h32, w32, self.cfg.pixel_decoder_feat_dim // 2))
        return self._consts[key]

    # ---- forward -------------------------------------------------------------------------------
    def _csp_run(self, packed, cat, out=None):
        both, reps = packed
        C = both.w.shape[0] // 2
        y12 = self._conv(both, cat, out_pair=True)
        x = _channels(y12, 0, C)
        for i, r in enumerate(reps):
            last = i == len(reps) - 1
            x = self._conv(r, x, residual=_channels(y12, C, 2 * C) if last else None, act=(ops.ACT_SILU | 16) if last else None, out=out if last else None,
                           out_pair=True)
        return x

    def _aifi(self, src, pos):
        """AIFI encoder layer (nn/layers/transformer.py:583-601, post-norm, GELU) on tokens [B,L,d] (fp32 under fp32_tc) -> (tokens, their operand)"""
        blk, d = self.aifi, src.shape[-1]
        sp, spp = self._with_pos(src, pos, want_op=True)
        qk = self._linear(blk["qk"], spp)
        v = self._linear(blk["v"], sp)
        a = ops.attention(qk[..., :d], qk[..., d:], v, self.nhead, 1.0 / math.sqrt(d // self.nhead), split=self.pair, out_pair=self.pair)
        x1, x1p, _ = self._norm(self._linear(blk["out"], a, residual=src), blk["n_attn"])
        if self.pair:  # no layer of the pair flow has a GELU epilogue: the split that writes linear2's operand applies it
            h, _ = ops.split_pair_ex(self._linear(blk["l1"], x1p), act=ops.ACT_GELU)
        else:
            h = self._linear(blk["l1"], x1p, act=ops.ACT_GELU)
        x2, x2p, _ = self._norm(self._linear(blk["l2"], h, residual=x1), blk["n_ffn"])
        return x2, x2p

    def _trunk(self, images, taps):
        """backbone + hybrid encoder + decoder input projection -> (memory [B,S,d] - a Pair under fp32_tc, else in the storage dtype -, shapes, constants)"""
        cfg = self.cfg
        _, res3, res4, res5 = self.trunk.run(images)
        B, h32, w32, _ = res5.shape
        K = self._constants(h32, w32)
        C = cfg.pixel_decoder_feat_dim
        dev = images.device
        cat1 = self._empty((B, h32 * 2, w32 * 2, 2 * C), dev)  # [up(lat0) | proj(res4)]
        cat2 = self._empty((B, h32 * 4, w32 * 4, 2 * C), dev)  # [up(lat1) | proj(res3)]
        cat3 = self._empty((B, h32 * 2, w32 * 2, 2 * C), dev)  # [down(fpn1) | lat1]
        cat4 = self._empty((B, h32, w32, 2 * C), dev)          # [down(pan0) | lat0]
        self._conv(self.enc_in[0], res3, out=_channels(cat2, C, 2 * C))
        self._conv(self.enc_in[1], res4, out=_channels(cat1, C, 2 * C))
        if self.aifi is None:  # no encoder layer (modelling.py:315): the projected res5 feeds lateral_convs.0, as a Pair in the pair flow
            lat_in = self._conv(self.enc_in[2], res5, out_pair=True)
        else:
            src = self._conv(self.enc_in[2], res5).reshape(B, h32 * w32, C)  # tokens for the AIFI block: fp32 in the pair flow (LayerNorm / attention work on fp32)
            # AIFI (modelling.py:315-324)
            src, src_p = self._aifi(src, K["pos"])
            p5 = src.reshape(B, h32, w32, C)
            lat_in = ops.Pair(src_p.buf.reshape(B, h32, w32, 2 * C)) if self.pair else p5  # the pair flow's conv reads the pair its LayerNorm wrote
            if taps is not None:
                taps["aifi"] = p5
        # top-down FPN (modelling.py:328-336)
        lat0 = self._conv(self.lateral[0], lat_in, out=_channels(cat4, C, 2 * C))
        ops.resize_bilinear(lat0, (h32 * 2, w32 * 2), out=_channels(cat1, 0, C))
        fpn0 = self._csp_run(self.fpn[0], cat1)
        lat1 = self._conv(self.lateral[1], fpn0, out=_channels(cat3, C, 2 * C))
        ops.resize_bilinear(lat1, (h32 * 4, w32 * 4), out=_channels(cat2, 0, C))
        fpn1 = self._csp_run(self.fpn[1], cat2)
        # bottom-up PAN (modelling.py:338-345)
        self._conv(self.down[0], ops.resize_bilinear(fpn1, (h32 * 2, w32 * 2)), out=_channels(cat3, 0, C))
        pan0 = self._csp_run(self.pan[0], cat3)
        self._conv(self.down[1], ops.resize_bilinear(pan0, (h32, w32)), out=_channels(cat4, 0, C))
        pan1 = self._csp_run(self.pan[1], cat4)
        enc_outs = [pan1, pan0, fpn1]  # outs[::-1] (modelling.py:347): 1/32, 1/16, 1/8
        if taps is not None:
            taps.update(res3=_unpair(res3), res4=_unpair(res4), res5=_unpair(res5), fpn0=_unpair(fpn0), fpn1=_unpair(fpn1), pan0=_unpair(pan0), pan1=_unpair(pan1))
        # predictor: memory [B, S, d] (modelling.py:1145-1167), each level written in place
        shapes = K["shapes"]
        memory = self._empty((B, sum(h * w for h, w in shapes), self.d), dev)
        buf = memory.buf if self.pair else memory
        start = 0
        for i, (f, (h, w)) in enumerate(zip(enc_outs, shapes)):
            lvl = buf[:, start:start + h * w].unflatten(1, (h, w))
            self._conv(self.dec_in[i], f, out=ops.Pair(lvl) if self.pair else lvl)
            start += h * w
        return memory, shapes, K

    @torch.no_grad()
    def forward(self, images: torch.Tensor, taps: Optional[dict] = None):
        """images [B,3,H,W] fp32 0..255 or [B,H,W,3] uint8 (H,W multiples of 32) -> (scores [B,Q,C] fp32, boxes xyxy [B,Q,4] fp32)."""
        B, H, W = self._input_size(images)
        if H % 32 or W % 32:
            # DETRProcessor resizes to im_size; the encoder buffers, anchors and positional constants are laid out for 1/8 and 1/16 maps of exactly 4x and
            # 2x the 1/32 map, so the engine takes multiples of 32 - resize or pad in the processor (image_size) for other inputs
            raise ValueError(f"focoos_b200: input size {H}x{W} is not a multiple of 32; resize/pad the image (e.g. ModelInfo.im_size) before the model")
        memory, shapes, K = self._trunk(images, taps)
        value_all = self._linear(self.value_all, memory)  # [B,S,6*d], layer i uses columns [i*d,(i+1)*d)
        # query selection (modelling.py:1191-1232)
        t = self._linear(self.enc_output, memory)
        return self._forward_head(t, value_all, memory, shapes, K, B, memory.shape[1], taps)

    def _forward_head(self, t, value_all, memory, shapes, K, B, S, taps):
        """query selection + decoder + head on the encoder memory (a Pair under fp32_tc).  t = enc_output.0(memory) BEFORE the valid-mask fill
        (modelling.py:1202-1207)."""
        cfg, d = self.cfg, self.d
        nq, ncls = cfg.num_queries, cfg.num_classes
        ln_w, ln_b = self.enc_output_ln
        if self.pair:
            # output_memory = LayerNorm(where(valid, t, bias)) only ever feeds the score head (as a pair) and the gathered rows (recomputed from t:
            # same arithmetic)
            _, om_pair, _ = ops.layernorm_ex(t, ln_w, ln_b, valid=K["valid"], fill=self.enc_output.bias, want_f32=False)
            scores = ops.linear_rowmax_pair(om_pair, self.enc_score.w3, self.enc_score.bias)
            _, topk_ind = ops.topk(scores, nq)
            tgt, tgt_op, _ = ops.layernorm_ex(t, ln_w, ln_b, gather=topk_ind, valid=K["valid"], fill=self.enc_output.bias)
        else:
            output_memory = ops.layernorm(ops.row_select(t, K["valid"], self.enc_output.bias), ln_w, ln_b)
            if self.precision == "fp16" and self.algo == ops.ALGO_AUTO:
                # only the per-anchor maximum is ever used in eval (modelling.py:1210-1214): the [B,S,365] fp32 logits (395 MB at bs=32) are never materialised
                scores = ops.linear_rowmax(output_memory, self.enc_score.w, self.enc_score.bias)
            else:
                cls_buf = torch.empty((B, S, (ncls + 7) // 8 * 8), dtype=torch.float32, device=t.device)
                self._linear(self.enc_score, output_memory, out=cls_buf[..., :ncls])
                scores = ops.rowmax(cls_buf[..., :ncls])
            _, topk_ind = ops.topk(scores, nq)
            tgt = tgt_op = ops.gather_rows(output_memory, topk_ind)
        ref_unact = ops.box_add_anchors(self._mlp(self.enc_bbox, tgt_op, out_dtype=torch.float32), K["anchors"], topk_ind)
        ref = ops.box_sigmoid(ref_unact)
        if taps is not None:
            taps.update(memory=_unpair(memory), enc_scores=scores, topk_ind=topk_ind, target=tgt, ref_unact=ref_unact)
        _, qp = self._refine(None, ref, False)
        scale = 1.0 / math.sqrt(d // self.nhead)
        L = len(self.dec)
        # decoder (modelling.py:969-1020, eval: logits only from the last layer)
        for i, blk in enumerate(self.dec):
            pos = self._linear(self.qpos[1], qp)
            _, tpp = self._with_pos(tgt, pos)
            qk = self._linear(blk["qk"], tpp)
            v = self._linear(blk["v"], tgt_op)
            a = ops.attention(qk[..., :d], qk[..., d:], v, self.nhead, scale, split=self.pair, out_pair=self.pair)
            tgt, _, tpp = self._norm(self._linear(blk["out"], a, residual=tgt), blk["n_attn"], pos=pos, want_op=False)
            oa = self._linear(blk["oa"], tpp, out_dtype=torch.float32)
            c = ops.msda(value_all[..., i * d:(i + 1) * d], oa, ref, shapes, NUM_POINTS, self.nhead, out_dtype=self.dt, out_pair=self.pair)
            tgt, tgt_op, _ = self._norm(self._linear(blk["cross_out"], c, residual=tgt), blk["n_cross"])
            y = self._linear(blk["l2"], self._linear(blk["l1"], tgt_op, act=ops.ACT_RELU, out_pair=True), residual=tgt)
            tgt, tgt_op, _ = self._norm(y, blk["n_ffn"])
            ref, qp = self._refine(self._mlp(blk["bbox"], tgt_op, out_dtype=torch.float32), ref, i == L - 1)
            if taps is not None:
                taps[f"dec{i}_out"] = tgt
                taps[f"dec{i}_ref"] = ref
        if self.pair:
            # class logits on the tensor cores into a 16-byte-padded row (TMA store pitch), then sigmoid into the dense [B,Q,C] scores
            lbuf = torch.empty((B, nq, self.dec_score.w.shape[0]), dtype=torch.float32, device=t.device)  # (ncls + 3) // 4 * 4 rows of the padded head
            logits = self._linear(self.dec_score, tgt_op, out=lbuf)[..., :ncls]
            scores = ops.sigmoid_rows(logits)
        else:
            logits = self._linear(self.dec_score, tgt, out_dtype=torch.float32, algo=ops.ALGO_SIMT)  # [B,Q,C] contiguous
            scores = ops.box_sigmoid(logits)
        if taps is not None:
            taps.update(pred_logits=logits, pred_boxes_cxcywh=ref)
        return scores, ops.box_cxcywh_to_xyxy(ref)

    def _refine(self, delta, ref, last):
        """(ref refined by delta, or ref itself for delta None; query_pos_head.layers.0 on those boxes, None when last).  fp32_tc writes both in one
        launch, the second as the Pair operand of query_pos_head.layers.1; fp16 / fp32 run the layer on the CUDA cores (K = 4)."""
        if self.pair:
            return ops.box_refine_qpos(delta, ref, None if last else self.qpos[0].w, None if last else self.qpos[0].bias)
        ref = ref if delta is None else ops.box_refine(delta, ref)
        return ref, None if last else self._linear(self.qpos[0], ref, act=ops.ACT_RELU, out_dtype=self.dt, algo=ops.ALGO_SIMT)


class FAIDetr(_EngineModel):
    """Drop-in for the reference `FAIDetr(BaseModelNN)` (modelling.py:1273): same constructor argument, same
    state_dict, `forward(images[, targets]) -> DETRModelOutput`."""

    engine_cls = DetrEngine

    def __init__(self, config: DETRConfig, precision: str = "fp16"):
        c = config
        super().__init__(c, precision,
                         Encoder(build_trunk(c.backbone_config), c.pixel_decoder_feat_dim, c.pixel_decoder_out_dim, c.pixel_decoder_nhead,
                                 c.pixel_decoder_dim_feedforward, c.pixel_decoder_num_encoder_layers),
                         TransformerPredictor(c.pixel_decoder_out_dim, c.num_classes, c.transformer_predictor_hidden_dim, c.num_queries,
                                              c.transformer_predictor_nhead, c.transformer_predictor_dec_layers, c.transformer_predictor_dim_feedforward))
        self.train_precision = None  # training arithmetic: None (follow `precision`), "fp32", "fp32_tc" or "amp" (see train_graph)
        self.sync_bn = False    # training: BatchNorm statistics over all data-parallel ranks (torch.nn.SyncBatchNorm, trainer/trainer.py:334); set by the trainer
        self.freeze_bn = False  # training: every BatchNorm as FrozenBatchNorm2d (TrainerArgs.freeze_bn, trainer/trainer.py:330)
        from .train_step import freeze_backbone_at, freeze_backbone_norm
        freeze_backbone_at(self, getattr(c.backbone_config, "freeze_at", -1), getattr(c.backbone_config, "num_stages", 4))  # resnet.py:221-224
        if getattr(c.backbone_config, "freeze_norm", False):  # resnet.py:226 (the registry configs ship freeze_norm=false)
            freeze_backbone_norm(self)

    def train(self, mode: bool = True):
        self._engine = None  # packed (BN-folded, re-parameterised) weights are rebuilt from the parameters at the next eval forward
        return super().train(mode)

    def check_trainable(self):
        """fine-tuning runs on the ResNet trunk only: the backward kernels of the STDC trunk (depthwise 3x3/s2, 3x3/s2 average pool, the concat-free
        CatBottleneck) are not built, so an STDC-trunk detector (fai-detr-m-coco) serves inference only"""
        if self.config.backbone_config.model_type != "resnet":
            raise NotImplementedError(f"focoos_b200 fine-tunes fai-detr on the ResNet trunk only: the {self.config.backbone_config.model_type!r} trunk's "
                                      "backward kernels are not built (inference runs)")

    def train_graph(self):
        """training-mode forward built from the autograd ops (fai_detr_train.py); fp32 storage, tensor-core split products by default"""
        self.check_trainable()
        from .fai_detr_train import DetrTrainGraph
        # train_precision: "amp" = one tensor-core product on fp16-rounded operands, fp32 accumulation / storage (the reference's torch.autocast(fp16) arithmetic,
        # trainer/trainer.py:735; the trainer sets it from TrainerArgs.amp_enabled); None = follow the inference precision (fp32-accurate products / CUDA-core fp32)
        prec = getattr(self, "train_precision", None) or ("fp32" if self.precision == "fp32" else "fp32_tc")
        if getattr(self, "_train_graph", None) is None or self._train_graph.prec != prec:
            self._train_graph = DetrTrainGraph(self, prec)
        return self._train_graph

    def criterion(self):
        """SetCriterion with the config's matcher / loss weights (modelling.py:1295-1316)"""
        if getattr(self, "_criterion", None) is None:
            from .criterion import BoxHungarianMatcher, SetCriterion
            c = self.config
            self._criterion = SetCriterion(
                num_classes=c.num_classes,
                matcher=BoxHungarianMatcher(cost_class=c.matcher_cost_class, cost_bbox=c.matcher_cost_bbox, cost_giou=c.matcher_cost_giou,
                                            use_focal_loss=c.matcher_use_focal_loss, alpha=c.matcher_alpha, gamma=c.matcher_gamma),
                weight_dict={"loss_vfl": c.weight_dict_loss_vfl, "loss_bbox": c.weight_dict_loss_bbox, "loss_giou": c.weight_dict_loss_giou},
                losses=c.criterion_losses, eos_coef=c.criterion_eos_coef, focal_alpha=c.criterion_focal_alpha, focal_gamma=c.criterion_focal_gamma,
                deep_supervision=c.criterion_deep_supervision)
        return self._criterion

    def forward(self, images: torch.Tensor, targets: list = [], taps: Optional[dict] = None) -> DETRModelOutput:
        self._check_device(images)
        if self.training:  # modelling.py:1354-1356: losses only, empty logits/boxes
            assert targets is not None and len(targets) > 0, "targets should not be None or empty - training mode"
            outputs = self.train_graph().forward(images)
            losses = self.criterion()({k: v for k, v in outputs.items() if not k.startswith("_")}, targets)
            if taps is not None:
                taps.update(outputs)
            return DETRModelOutput(logits=torch.zeros(0, 0, 0), boxes=torch.zeros(0, 0, 4), loss=losses)
        scores, boxes = self.engine().forward(images if images.dtype == torch.uint8 else images.to(torch.float32), taps)
        return DETRModelOutput(boxes=boxes, logits=scores, loss=None)
