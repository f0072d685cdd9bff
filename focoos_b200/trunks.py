"""The conv trunks every model family runs on: ResNet-vd and STDC.  The parameter containers mirror the reference's module trees (same attribute names,
same parameter shapes, so a reference state_dict loads unchanged); `build_trunk` picks one from `backbone_config.model_type`.  `pack_trunk` packs the
same trunk for an engine (folded BN, fused NHWC convs): the packed trunk's `run(images)` gives [res2, res3, res4, res5] and its `pair_layers()` the
layers the fp32_tc flow runs on weight triples."""
import weakref
from collections import OrderedDict

import torch
import torch.nn as nn

from . import ops
from .engine import _bn_fold, _channels, _packed_layers
from .ports import ResnetConfig, STDCConfig

RESNET_BLOCKS = {50: [3, 4, 6, 3], 101: [3, 4, 23, 3]}


class ConvNormLayer(nn.Module):  # nn/layers/conv.py:78
    def __init__(self, ch_in, ch_out, k, stride, act=None):
        super().__init__()
        self.conv = nn.Conv2d(ch_in, ch_out, k, stride, padding=(k - 1) // 2, bias=False)
        self.norm = nn.BatchNorm2d(ch_out)
        self.act_name, self.stride = act, stride


class BottleNeck(nn.Module):  # nn/backbone/resnet.py:72
    def __init__(self, ch_in, ch_out, stride, shortcut):
        super().__init__()
        self.branch2a = ConvNormLayer(ch_in, ch_out, 1, 1, "relu")
        self.branch2b = ConvNormLayer(ch_out, ch_out, 3, stride, "relu")
        self.branch2c = ConvNormLayer(ch_out, ch_out * 4, 1, 1)
        self.shortcut, self.stride = shortcut, stride
        if not shortcut:
            if stride == 2:
                self.short = nn.Sequential(OrderedDict([("pool", nn.AvgPool2d(2, 2, 0, ceil_mode=True)), ("conv", ConvNormLayer(ch_in, ch_out * 4, 1, 1))]))
            else:
                self.short = ConvNormLayer(ch_in, ch_out * 4, 1, stride)


class Blocks(nn.Module):  # nn/backbone/resnet.py:124
    def __init__(self, ch_in, ch_out, count, stage_num):
        super().__init__()
        self.blocks = nn.ModuleList()
        for i in range(count):
            self.blocks.append(BottleNeck(ch_in, ch_out, stride=2 if i == 0 and stage_num != 2 else 1, shortcut=i != 0))
            if i == 0:
                ch_in = ch_out * 4


class ResNet(nn.Module):  # nn/backbone/resnet.py:164 (variant d, depth >= 50)
    def __init__(self, cfg: ResnetConfig):
        super().__init__()
        assert cfg.variant == "d" and cfg.depth in RESNET_BLOCKS, "focoos_b200 implements ResNet-50/101 vd"
        self.depth = cfg.depth
        self.conv1 = nn.Sequential(OrderedDict([
            ("conv1_1", ConvNormLayer(cfg.in_chans, 32, 3, 2, "relu")),
            ("conv1_2", ConvNormLayer(32, 32, 3, 1, "relu")),
            ("conv1_3", ConvNormLayer(32, 64, 3, 1, "relu")),
        ]))
        self.res_layers = nn.ModuleList()
        ch_in = 64
        for i, (n, ch) in enumerate(zip(RESNET_BLOCKS[cfg.depth], [64, 128, 256, 512])):
            self.res_layers.append(Blocks(ch_in, ch, n, i + 2))
            ch_in = ch * 4
        self.out_channels = [256, 512, 1024, 2048]


class ConvX(nn.Module):  # nn/backbone/stdc.py:20 — also ConvBNReLU (bisenetformer/modelling.py:122)
    def __init__(self, cin, cout, k=3, stride=1):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride, padding=k // 2, bias=False)
        self.bn = nn.BatchNorm2d(cout)


class CatBottleneck(nn.Module):  # nn/backbone/stdc.py:109
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.stride = stride
        if stride == 2:
            self.avd_layer = nn.Sequential(nn.Conv2d(cout // 2, cout // 2, 3, 2, 1, groups=cout // 2, bias=False), nn.BatchNorm2d(cout // 2))
        self.conv_list = nn.ModuleList([ConvX(cin, cout // 2, 1), ConvX(cout // 2, cout // 4), ConvX(cout // 4, cout // 8), ConvX(cout // 8, cout // 8)])


class STDC(nn.Module):  # nn/backbone/stdc.py:189
    def __init__(self, cfg: STDCConfig):
        super().__init__()
        assert cfg.block_type == "cat" and cfg.block_num == 4, "focoos_b200 implements the CatBottleneck STDC (block_num 4)"
        base, feats = cfg.base, []
        feats += [ConvX(cfg.in_chans, base // 2, 3, 2), ConvX(base // 2, base, 3, 2)]
        for i, n in enumerate(cfg.layers):
            for j in range(n):
                if i == 0 and j == 0:
                    feats.append(CatBottleneck(base, base * 4, 2))
                elif j == 0:
                    feats.append(CatBottleneck(base * 2 ** (i + 1), base * 2 ** (i + 2), 2))
                else:
                    feats.append(CatBottleneck(base * 2 ** (i + 2), base * 2 ** (i + 2), 1))
        self.features = nn.Sequential(*feats)
        self.out_channels = [base, base * 4, base * 8, base * 16]


class _PackedTrunk:
    """a trunk packed by its engine's `_pack_conv` and run through its engine's `_conv`; `stem` is the fp32 first conv that ops.stem_conv runs with the
    input normalisation"""

    def __init__(self, eng):
        self.eng = weakref.proxy(eng)  # the engine owns the trunk: no reference cycle keeps a dropped engine's device weights alive

    def pair_layers(self):
        """every layer but the stem"""
        return [layer for layer in _packed_layers(vars(self)) if layer is not self.stem]

    def _stem(self, images, out_pair=False):
        eng = self.eng
        return ops.stem_conv(images.contiguous(), self.stem.w, self.stem.scale, self.stem.bias, eng.cfg.pixel_mean, eng.cfg.pixel_std, ops.ACT_RELU, eng.dt,
                             out_pair=out_pair)


class ResNetTrunk(_PackedTrunk):
    """ResNet-vd (nn/backbone/resnet.py:164): stem + bottleneck stages."""

    def __init__(self, eng, sd, bb):
        super().__init__(eng)
        cnl = lambda p, act=ops.ACT_RELU, stride=1, dtype=None: eng._pack_conv(sd, p + ".conv.weight", bn=p + ".norm", stride=stride, act=act, dtype=dtype)
        self.stem = cnl(bb + ".conv1.conv1_1", stride=2, dtype=torch.float32)
        self.stem2, self.stem3 = cnl(bb + ".conv1.conv1_2"), cnl(bb + ".conv1.conv1_3")
        self.stages = []
        for si, count in enumerate(RESNET_BLOCKS[eng.cfg.backbone_config.depth]):
            blocks = []
            for bi in range(count):
                p = f"{bb}.res_layers.{si}.blocks.{bi}"
                stride = 2 if (bi == 0 and si != 0) else 1
                blk = {"a": cnl(p + ".branch2a"), "b": cnl(p + ".branch2b", stride=stride), "c": cnl(p + ".branch2c"), "stride": stride, "short": None}
                if bi == 0:
                    blk["short"] = cnl(p + (".short.conv" if stride == 2 else ".short"), ops.ACT_NONE)
                blocks.append(blk)
            self.stages.append(blocks)

    def run(self, images):
        """nn/backbone/resnet.py:252-266: Pairs under fp32_tc"""
        conv = self.eng._conv
        x = conv(self.stem3, conv(self.stem2, self._stem(images, out_pair=self.eng.pair), out_pair=True), out_pair=True)
        x = ops.maxpool3x3s2(x)
        feats = []
        for blocks in self.stages:
            for blk in blocks:
                y = conv(blk["b"], conv(blk["a"], x, out_pair=True), out_pair=True)
                short = x if blk["short"] is None else conv(blk["short"], ops.avgpool2x2(x) if blk["stride"] == 2 else x, out_pair=True)
                x = conv(blk["c"], y, residual=short, out_pair=True)
            feats.append(x)
        return feats


class STDCTrunk(_PackedTrunk):
    """STDC (nn/backbone/stdc.py:189): two stride-2 ConvX stems + CatBottleneck stages; stride-2 blocks keep the depthwise 3x3/s2 + BN weights fp32 [9, C]."""

    def __init__(self, eng, sd, bb):
        super().__init__(eng)
        bb += ".features"
        convx = lambda p, stride=1, dtype=None: eng._pack_conv(sd, p + ".conv.weight", bn=p + ".bn", stride=stride, act=ops.ACT_RELU, dtype=dtype)
        self.stem = convx(bb + ".0", 2, torch.float32)
        self.stem2 = convx(bb + ".1", 2)
        self.blocks = []
        idx = 2
        for n in eng.cfg.backbone_config.layers:
            stage = []
            for j in range(n):
                p = f"{bb}.{idx}"
                stride = 2 if j == 0 else 1
                blk = {"stride": stride, "convs": [convx(f"{p}.conv_list.{i}") for i in range(4)]}
                if stride == 2:
                    wd = sd[p + ".avd_layer.0.weight"].float()  # [C,1,3,3]
                    sa, ba = _bn_fold(sd, p + ".avd_layer.1")
                    blk["avd"] = (eng._f32(wd.reshape(wd.shape[0], 9).t()), eng._f32(sa), eng._f32(ba))
                stage.append(blk)
                idx += 1
            self.blocks.append(stage)

    def run(self, images):
        """nn/backbone/stdc.py:314: res2 fp32 under fp32_tc; res3-5 are Pairs where the stage's last block runs in the pair format (_pair_block_ok)"""
        x = self.eng._conv(self.stem2, self._stem(images))  # res2
        feats = [x]
        for stage in self.blocks:
            for blk in stage:
                x = self._cat_bottleneck(x, blk)
            feats.append(x)
        return feats

    def _cat_bottleneck(self, x, blk):
        """CatBottleneck, concat-free: each conv writes its channel slice of the block's output buffer, which the next conv reads in place.  A block that
        _pair_block_ok takes keeps the buffer as a Pair (no split pass inside the block); a stride-2 block's first conv reads a Pair input and writes fp32."""
        conv, dt = self.eng._conv, self.eng.dt
        c = blk["convs"]
        half = c[0].w.shape[0]
        B, H, W, _ = x.shape
        if blk["stride"] == 2:
            out1 = conv(c[0], x)
            buf = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 2 * half), dtype=dt, device=x.device)
            ops.avgpool3x3s2(out1, out=buf[..., :half])
            src = ops.dwconv3x3s2(out1, *blk["avd"])
        else:
            shape = (B, H, W, 2 * half)
            buf = ops.Pair.empty(shape, x.device) if self._pair_block_ok(blk, H, W) else torch.empty(shape, dtype=dt, device=x.device)
            src = conv(c[0], x, out=_channels(buf, 0, half))
        o = half
        for i in (1, 2, 3):
            w = c[i].w.shape[0]
            src = conv(c[i], src, out=_channels(buf, o, o + w))
            o += w
        return buf

    def _pair_block_ok(self, blk, H, W) -> bool:
        """conv2d_pair takes the block: every conv has its weight triple; a 32-channel 3x3 input needs the halo mode (rows of at least 64 pixels, Cout <= 64)"""
        if blk["stride"] != 1 or not self.eng.pair:
            return False
        for cv in blk["convs"]:
            cin, cout, k = cv.w.shape[3], cv.w.shape[0], cv.w.shape[1]
            if cv.w3 is None or cout % 8:
                return False
            if cin % 64 and not (cin == 32 and k == 3 and W >= 64 and cout <= 64):
                return False
        return True


_TRUNKS = {"resnet": (ResNet, ResNetTrunk), "stdc": (STDC, STDCTrunk)}


def build_trunk(backbone_config):
    """the parameter container of the trunk that backbone_config.model_type names"""
    return _TRUNKS[backbone_config.model_type][0](backbone_config)


def pack_trunk(eng, sd, bb="pixel_decoder.backbone"):
    """the trunk of eng.cfg under state_dict prefix `bb`, packed for the engine `eng`"""
    return _TRUNKS[eng.cfg.backbone_config.model_type][1](eng, sd, bb)
