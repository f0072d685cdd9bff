"""The family-neutral side of every inference engine: packed layers, host-side packing, the layer call that picks a conv / linear kernel, and the
nn.Module lifecycle (`_EngineModel`) the model classes share.  The engines of the families (fai_detr.DetrEngine, fai_mf.MFEngine,
bisenetformer.BisenetEngine) subclass `Engine` and write their own `_pack`, `_pair_layers` and `forward`; the conv trunks they run on are in trunks.py."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from . import ops


def _split3_weights(w):
    """fp32 [..., C] -> fp16 [..., 3C] = [W_hi | W_lo | W_hi] (the weight operand of fb200_conv2d_pair)."""
    hi = w.half()
    lo = (w - hi.float()).half()
    return torch.cat([hi, lo, hi], dim=-1).contiguous()


class _Conv:
    """Packed conv: weight [Cout,KH,KW,Cin] in activation dtype, fp32 scale/bias (folded BN).
    `w3` (precision="fp32_tc"): the [W_hi|W_lo|W_hi] fp16 triple of the pair flow's tensor-core products.  Run by Engine._conv."""

    __slots__ = ("w", "scale", "bias", "stride", "pad", "act", "w3")

    def __init__(self, w, scale, bias, stride=1, pad=0, act=ops.ACT_NONE):
        self.w, self.scale, self.bias, self.stride, self.pad, self.act, self.w3 = w, scale, bias, stride, pad, act, None


class _Linear:
    """Packed linear: weight [N,K] in activation dtype, fp32 bias, `w3` as in _Conv.  Run by Engine._linear."""

    __slots__ = ("w", "bias", "w3")

    def __init__(self, w, bias):
        self.w, self.bias, self.w3 = w, bias, None


def _pad_rows(lin, mult):
    """a packed linear with zero output rows (weight, weight triple, bias) up to a multiple of `mult`"""
    n = -lin.w.shape[0] % mult
    if not n:
        return lin
    pad = lambda t: torch.cat([t, t.new_zeros((n, *t.shape[1:]))])
    out = _Linear(pad(lin.w), pad(lin.bias))
    out.w3 = pad(lin.w3)
    return out


def _unpair(t):
    """a Pair as its fp32 values (a torch op: taps and the small 1/32 map of BisenetFormer's context path), any tensor as it is"""
    return t.float() if isinstance(t, ops.Pair) else t


def _channels(t, a, b):
    """channels [a, b) of an NHWC activation buffer (a tensor view or a Pair slice): concat-free blocks write their branches into them"""
    return t.slice(a, b) if isinstance(t, ops.Pair) else t[..., a:b]


_PAIR_MIN_ROWS = 64  # fp32_tc: an fp32 operand with fewer rows (MaskFormer's 1/32 encoder below ~256x256 input) stays on the CUDA-core fp32 kernel


def _packed_layers(obj, seen=None):
    """every packed layer (_Conv / _Linear) reachable from obj through dicts / lists / tuples and packed trunks (trunks.py), once each"""
    seen = set() if seen is None else seen
    if id(obj) in seen:
        return
    seen.add(id(obj))
    if isinstance(obj, (_Conv, _Linear)):
        yield obj
    elif isinstance(obj, dict):
        for v in obj.values():
            yield from _packed_layers(v, seen)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            yield from _packed_layers(v, seen)
    elif hasattr(obj, "pair_layers"):  # a packed trunk: its layers are its attributes
        yield from _packed_layers(vars(obj), seen)


def _bn_fold(sd, p, eps=1e-5):
    s = sd[p + ".weight"].float() / torch.sqrt(sd[p + ".running_var"].float() + eps)
    return s, sd[p + ".bias"].float() - sd[p + ".running_mean"].float() * s


class Engine:
    """Packs a state_dict for one (device, precision) and runs the fused forward.  A family's engine implements `_pack` (its packed layers as
    attributes), `_pair_layers` (the packed layers the fp32_tc flow runs on their weight triples) and `forward`.

    precision "fp16" / "fp32": activations in that dtype; `algo` goes to every conv / linear (ALGO_SIMT: the CUDA-core kernels).
    precision "fp32_tc": the pair flow - fp32 storage, every conv / linear of the flow three fp16 tensor-core products on activations kept as fp16 [hi | lo]
    planes between them; it runs only with the default algorithm choice.  `_conv` / `_linear` pick the kernel of every layer."""

    def __init__(self, sd: Dict[str, torch.Tensor], cfg, device, precision: str = "fp16", algo: int = ops.ALGO_AUTO):
        assert precision in ("fp32", "fp16", "fp32_tc")
        if precision == "fp32_tc" and algo != ops.ALGO_AUTO:
            raise ValueError(f"focoos_b200: precision 'fp32_tc' runs the tensor-core pair flow and takes no other algorithm (got algo={algo})")
        self.cfg, self.device, self.precision, self.algo = cfg, torch.device(device), precision, algo
        self.pair = precision == "fp32_tc"
        self.dt = torch.float16 if precision == "fp16" else torch.float32
        self._consts = {}  # per-resolution constants (DetrEngine._constants, MFEngine._pos)
        self._host_w3 = {} if self.pair else None  # id(packed device weight) -> [W_hi|W_lo|W_hi] split on the host in _to()
        # pack on the HOST (BN folding, re-parameterisation, concatenations are a few hundred tiny tensor ops: as device launches they were ~700 `at::`
        # kernels in front of the first forward); only the packed tensors travel to the device
        sd = {k: v.detach().to("cpu") for k, v in sd.items()}
        self._pack(sd)
        if self.pair:
            for layer in _packed_layers(vars(self)):
                if layer.w.dtype == torch.float32 and layer.w.shape[-1] % 32 == 0:
                    layer.w3 = self._host_w3.get(id(layer.w))
                    if layer.w3 is None:
                        layer.w3 = _split3_weights(layer.w)
            assert all(layer.w3 is not None for layer in self._pair_layers()), "fp32_tc: a layer of the pair flow has no [W_hi|W_lo|W_hi] weight triple"
        self._host_w3 = None

    @staticmethod
    def _input_size(images):
        """B, H, W of the images: uint8 NHWC [B,H,W,3] (decoded images, straight into the stem kernel) or fp32 NCHW [B,3,H,W] 0..255"""
        if images.dtype == torch.uint8:
            assert images.dim() == 4 and images.shape[3] == 3
            return images.shape[0], images.shape[1], images.shape[2]
        assert images.dim() == 4 and images.shape[1] == 3 and images.dtype == torch.float32
        return images.shape[0], images.shape[2], images.shape[3]

    # ---- packing -------------------------------------------------------------------------------
    def _to(self, t, dtype=None):
        d = t.to(device=self.device, dtype=dtype or self.dt).contiguous()
        if self._host_w3 is not None and dtype is None and t.dim() >= 2 and t.shape[-1] % 32 == 0 and not t.is_cuda:
            self._host_w3[id(d)] = _split3_weights(t.float().contiguous()).to(self.device)
        return d

    def _f32(self, t):
        return t.to(device=self.device, dtype=torch.float32).contiguous()

    def _pack_conv(self, sd, w, bn=None, bias=None, stride=1, act=ops.ACT_NONE, dtype=None):
        """the state_dict conv weight `w` (key) -> _Conv with padding k // 2: the BatchNorm at key prefix `bn` folded into the epilogue's scale / bias, or
        the conv's own `bias` (key), or neither.  The weight is stored in the activation dtype unless `dtype` says otherwise."""
        wt = sd[w].float()
        scale, shift = _bn_fold(sd, bn) if bn is not None else (None, None if bias is None else sd[bias])
        f32 = lambda t: None if t is None else self._f32(t)
        return _Conv(self._to(wt.permute(0, 2, 3, 1), dtype), f32(scale), f32(shift), stride, wt.shape[-1] // 2, act)

    def _lin(self, sd, p, dtype=None):
        return _Linear(self._to(sd[p + ".weight"].float(), dtype), self._f32(sd[p + ".bias"].float()))

    def _pack_attn_block(self, sd, p, ffn_norms, d=None):
        """MultiheadAttention (packed in_proj: rows [0,d)=Q, [d,2d)=K, [2d,3d)=V) + FFN + the two LayerNorms around them; d defaults to self.d."""
        d = self.d if d is None else d
        w, b = sd[p + ".self_attn.in_proj_weight"].float(), sd[p + ".self_attn.in_proj_bias"].float()
        n_attn, n_ffn = ffn_norms
        return {
            "qk": _Linear(self._to(w[: 2 * d]), self._f32(b[: 2 * d])), "v": _Linear(self._to(w[2 * d:]), self._f32(b[2 * d:])),
            "out": self._lin(sd, p + ".self_attn.out_proj"), "l1": self._lin(sd, p + ".linear1"), "l2": self._lin(sd, p + ".linear2"),
            "n_attn": (self._f32(sd[f"{p}.{n_attn}.weight"]), self._f32(sd[f"{p}.{n_attn}.bias"])),
            "n_ffn": (self._f32(sd[f"{p}.{n_ffn}.weight"]), self._f32(sd[f"{p}.{n_ffn}.bias"])),
        }

    # ---- the layer call: the one place that picks a conv / linear kernel from the precision and the operand's format ---------------------------------
    def _on_pairs(self, layer, x, algo, out_pair):
        """fp32_tc: whether the layer runs as three fp16 tensor-core products on the pair planes of x (conv2d_pair) rather than on the fp32 CUDA cores.
        A Pair operand or a Pair result can only take the products.  An fp32 operand with an fp32 result stays on the CUDA cores when the call asks for
        ALGO_SIMT (the [B,C] gates, the MaskFormer classifier), when the layer has no weight triple, or when it has fewer than _PAIR_MIN_ROWS rows."""
        if not self.pair:
            return False
        if isinstance(x, ops.Pair) or out_pair:
            return True
        return algo != ops.ALGO_SIMT and layer.w3 is not None and x.numel() // x.shape[-1] >= _PAIR_MIN_ROWS

    def _conv(self, conv, x, *, act=None, residual=None, out=None, out_dtype=None, algo=None, out_pair=False):
        """one packed conv.  fp16 / fp32: ops.conv2d on the storage weight with `algo` (default self.algo).  fp32_tc (see _on_pairs): ops.conv2d_pair on
        the weight triple - x a Pair or split into one - whose result is a Pair with out_pair=True or a Pair `out`, else fp32.  The storage flow ignores
        out_pair.  The residual has the result's format."""
        act = conv.act if act is None else act
        algo = self.algo if algo is None else algo
        if self._on_pairs(conv, x, algo, out_pair or isinstance(out, ops.Pair)):
            assert act & 15 not in (ops.ACT_GELU, ops.ACT_SIGMOID), "no layer of the pair flow has a GELU / sigmoid epilogue"
            return ops.conv2d_pair(ops.to_pair(x), conv.w3, conv.scale, conv.bias, stride=conv.stride, pad=conv.pad, act=act, residual=residual, out=out,
                                   out_pair=out_pair)
        return ops.conv2d(x, conv.w, conv.scale, conv.bias, stride=conv.stride, pad=conv.pad, act=act, residual=residual, out=out, out_dtype=out_dtype, algo=algo)

    def _linear(self, lin, x, *, act=ops.ACT_NONE, residual=None, out=None, out_dtype=None, algo=None, out_pair=False):
        """one packed linear on tokens [..., K]: ops.linear, or under fp32_tc ops.linear_pair, chosen as in _conv.  `out` may be a column slice of a wider
        fp32 buffer."""
        algo = self.algo if algo is None else algo
        if self._on_pairs(lin, x, algo, out_pair):
            assert act & 15 not in (ops.ACT_GELU, ops.ACT_SIGMOID), "no layer of the pair flow has a GELU / sigmoid epilogue"
            return ops.linear_pair(ops.to_pair(x), lin.w3, lin.bias, act=act, residual=residual, out=out, out_pair=out_pair)
        return ops.linear(x, lin.w, lin.bias, act=act, residual=residual, out=out, out_dtype=out_dtype, algo=algo)

    # ---- the row glue between two linears of the transformer layers: the one place that picks it from the precision --------------------------------------
    # fp32_tc: the fused glue kernels (csrc/head_fused.cu) - LayerNorm, positional add, GELU - write the Pair operand of the next tensor-core linear
    # themselves, so no separate split / add launch sits between two linears.  fp16 / fp32: ops.layernorm / ops.add in the storage dtype.
    def _operand(self, x):
        """x as a linear operand of the flow: its Pair under fp32_tc (one split launch), else x"""
        return ops.to_pair(x) if self.pair else x

    def _with_pos(self, x, pos, want_op=False):
        """(x as an operand if want_op else None, x + pos as an operand); fp32_tc writes both in one launch"""
        if self.pair:
            return ops.split_pair_ex(x, pos=pos, want_pair=want_op, want_pair_pos=True)
        return (x if want_op else None), ops.add(x, pos)

    def _norm(self, y, ln, *, pos=None, want_f32=True, want_op=True):
        """x = LayerNorm(y) with ln = (gamma, beta) -> (x, x as an operand, x + pos as an operand or None without pos); fp32_tc writes them in one launch.
        want_f32 / want_op let fp32_tc skip an output no one reads (None in its place); the storage flow returns its one tensor in both places."""
        if self.pair:
            return ops.layernorm_ex(y, *ln, pos=pos, want_f32=want_f32, want_pair=want_op, want_pair_pos=pos is not None)
        x = ops.layernorm(y, *ln)
        return x, x, (None if pos is None else ops.add(x, pos))

    def _mlp(self, layers, x, out_dtype=None):
        """packed linears with ReLU between them; under fp32_tc the hidden activations stay Pairs"""
        for lin in layers[:-1]:
            x = self._linear(lin, x, act=ops.ACT_RELU, out_pair=True)
        return self._linear(layers[-1], x, out_dtype=out_dtype)

    def _empty(self, shape, device):
        """an activation buffer of the flow: a Pair under fp32_tc, else a tensor in the storage dtype"""
        return ops.Pair.empty(shape, device) if self.pair else torch.empty(shape, dtype=self.dt, device=device)


class _Head(nn.Module):
    """`head` of every family (the reference's DETRHead / MaskFormerHead / BisenetFormerHead): the predictor, and `criterion.empty_weight`, which
    is in the weight file (SURVEY Appendix B) though inference computes no loss"""

    def __init__(self, predictor, num_classes):
        super().__init__()
        w = torch.ones(num_classes + 1)
        w[-1] = 0.1
        self.criterion = nn.Module()
        self.criterion.register_buffer("empty_weight", w)
        self.predictor = predictor


class _EngineModel(nn.Module):
    """The nn.Module side of every model family: parameters under the reference's state_dict keys (`pixel_decoder`, then `head`: `predictor`), `.device` /
    `.dtype` from the non-persistent `pixel_mean` buffer, and the `engine_cls` engine packed from the parameters for the current (device, precision,
    algo) on first use, dropped whenever they may change.  A model starts in eval mode."""

    engine_cls: type

    def __init__(self, config, precision: str, pixel_decoder: nn.Module, predictor: nn.Module):
        super().__init__()
        self.config, self.num_classes, self.precision, self.algo, self._engine = config, config.num_classes, precision, ops.ALGO_AUTO, None
        self.pixel_decoder, self.head = pixel_decoder, _Head(predictor, config.num_classes)
        self.register_buffer("pixel_mean", torch.tensor(config.pixel_mean, dtype=torch.float32).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor(config.pixel_std, dtype=torch.float32).view(-1, 1, 1), False)
        self.eval()

    device = property(lambda self: self.pixel_mean.device)
    dtype = property(lambda self: self.pixel_mean.dtype)

    def load_state_dict(self, state_dict, strict: bool = False, assign: bool = False):
        """Shape-tolerant non-strict load like BaseModelNN.load_state_dict (models/base_model.py:98-143); accepts
        {"model": sd} checkpoints (focoos_model.py:684-685)."""
        if "model" in state_dict and isinstance(state_dict["model"], dict):
            state_dict = state_dict["model"]
        own = self.state_dict()
        filtered = {k: v for k, v in state_dict.items() if k in own and tuple(own[k].shape) == tuple(v.shape)}
        res = super().load_state_dict(filtered, strict=False)
        self._engine = None
        if strict and (res.missing_keys or len(filtered) != len(state_dict)):
            raise RuntimeError(f"load_state_dict(strict): missing {res.missing_keys[:5]} / dropped {len(state_dict) - len(filtered)}")
        return res

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def engine(self):
        e = self._engine
        if e is None or e.device != self.device or e.precision != self.precision or e.algo != self.algo:
            self._engine = self.engine_cls(self.state_dict(), self.config, self.device, self.precision, self.algo)
        return self._engine

    def _check_device(self, images):
        if ops._backend is None and not images.is_cuda:
            raise RuntimeError(f"focoos_b200.{type(self).__name__} runs on CUDA (sm_90a) only — no CPU fallback; move the model and inputs to the GPU")
