"""Per-launch fp64 check of every conv / linear kernel launch a model makes (test infrastructure, not a conftest).

`CheckingBackend(inner)` stands in for `ops._backend`: it wraps conv2d, conv2d_pair, linear_rowmax, linear_rowmax_pair, stem_conv and dwconv3x3s2 of
`inner` (the CUDA backend, or the CPU reference backend) and passes every other operator through.  For each wrapped call it snapshots the exact operand
values the launch receives (a Pair counts as hi + lo, a weight triple [W_hi | W_lo | W_hi] as W_hi + W_lo, fp16 operands as they are), runs the launch,
and compares the result with plain torch in float64 on the same operands (folded scale / bias, residual before or after the activation, per-image
weights, the row maximum).  Because each launch is compared with its own operands, the chaos a seeded decoder shows end to end (discrete attention-mask
bits flipping on 1e-5 differences) does not reach the comparison, and the bars stay where the arithmetic puts them:

  1. per element   |y - y64| <= bound                      (tile edges, channel tails, slices, taps)
  2. per launch    ||y - y64||_2 <= ||agg_bound||_2        (a precision loss spread thin: a dropped lo plane or hi x W_lo product)
  3. a Pair output encodes its value: hi is a nearest fp16 of hi + lo (|lo| <= half the fp16 gap from hi towards lo)
  4. nothing in the output's storage span (first to last element, plus one pixel pitch each side) outside the output view changed
  5. the inputs are unchanged, unless they share storage with the output (that part of them is then covered by 4)

Check 3 allows the tie: hi = fp16(v), lo = fp16(v - hi) can round lo up to exactly half an fp16 ulp of hi, and fp16(hi + lo) then rounds to even, away
from hi, for about one element in 6000.  That is a correct split, so "hi == fp16(hi + lo)" alone would reject it.
"""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.nn.functional as F

from focoos_b200.ops import Pair

# ---- the bounds, from unit roundoff ------------------------------------------------------------------------------------------------------------------
# A = |s| * conv(|x|, |w|) + |b| (+ |r|) in fp64 is the magnitude of the terms a launch sums.  With K products per output:
#   bound = LIP * ((C_ACC * sqrt(K) + C_EPI) * u32 + LOLO[arith]) * A  +  (C_OUT * u32 + FMT[fmt].rel) * |y64|  +  FMT[fmt].abs
U32 = 2.0 ** -24  # unit roundoff of fp32
C_ACC = 4.0       # fp32 accumulation of K terms: the probabilistic bound sqrt(K) * u32 * A (Higham & Mary), with a margin of 4 for the worst of ~1e8 elements
C_EPI = 4.0       # the fp32 epilogue: scale, bias, residual add (and the stem's image normalisation), a few roundings of values below A
C_OUT = 4.0       # the activation's own evaluation (expf / erff), relative to its result
LIP = 1.13        # largest slope of the activations: ReLU 1, SiLU 1.10, exact-erf GELU 1.13, sigmoid 0.25 - the pre-activation error carries through
C_AGG = 8.0       # per launch, the accumulation term without sqrt(K): products of either sign make the partial sums a random walk whose rounding
                  # errors cancel to O(u32 * A) per element, so a systematic loss of 2^-20 of A over a whole launch stands out
# split products (fp32_tc) omit lo x W_lo: |lo| <= 2^-11 |x| and |W_lo| <= 2^-11 |w|, so at most 2^-22 of every product
LOLO = {"fp32": 0.0, "fp16": 0.0, "split": 2.0 ** -22}
# output format: (relative, absolute) rounding of the stored result.  fp16 rounds to 2^-11 |y|; a Pair keeps v - hi to 2^-11, i.e. 2^-22 |y|.  Both
# lose up to half the smallest fp16 subnormal (2^-25) where the value (fp16) or v - hi (Pair) falls below 2^-14.
FMT = {"fp32": (0.0, 0.0), "fp16": (2.0 ** -11, 2.0 ** -25), "pair": (2.0 ** -22, 2.0 ** -25)}


def _site():
    """file:function:line of the model code that made the launch: the first frame outside the operator layer, this module and the engines' generic
    layer calls (_conv / _linear)"""
    f = sys._getframe(2)
    skip = (os.sep + "ops.py", os.sep + "conv_launch_check.py")
    while f is not None and (f.f_code.co_filename.endswith(skip) or f.f_code.co_name in ("_conv", "_linear")):
        f = f.f_back
    if f is None:
        return "?"
    return f"{os.path.basename(f.f_code.co_filename)}:{f.f_code.co_name}:{f.f_lineno}"


def _val64(t):
    """the fp64 values of an operand as the launch receives it (a Pair: hi + lo); a new tensor, so it is a snapshot"""
    if t is None:
        return None
    if isinstance(t, Pair):
        return t.hi.double() + t.lo.double()
    return t.double()


def _views(t):
    """the tensor views an operand or output occupies (a Pair: its hi and lo planes)"""
    if t is None:
        return []
    return [t.hi, t.lo] if isinstance(t, Pair) else [t]


def _extent(v):
    """(first, last) element offset of a view in its storage"""
    first = v.storage_offset()
    return first, first + sum((n - 1) * s for n, s in zip(v.shape, v.stride()))


def _flat(v):
    """the whole storage of a view as a 1-D tensor of its dtype"""
    n = v.untyped_storage().nbytes() // v.element_size()
    return torch.empty(0, dtype=v.dtype, device=v.device).set_(v.untyped_storage(), 0, (n,), (1,))


_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _bits(t):
    return t.contiguous().view(_INT[t.element_size()]) if t.dtype.is_floating_point else t.contiguous()


def _act64(z, act):
    a = act & 15
    if a == 1:
        return torch.relu(z)
    if a == 2:
        return z * torch.sigmoid(z)
    if a == 3:
        return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))
    if a == 4:
        return torch.sigmoid(z)
    assert a == 0, f"unknown activation {act}"
    return z


def _conv64(x, w, stride, pad, groups=1):
    """NHWC fp64 conv; w [Cout,KH,KW,Cin], or [B,Cout,KH,KW,Cin] with one weight set per image"""
    if w.dim() == 5:
        if w.shape[2] == 1 and w.shape[3] == 1 and stride == 1:
            return torch.einsum("bhwc,bqc->bhwq", x, w[:, :, 0, 0])
        B = x.shape[0]
        xn = x.permute(0, 3, 1, 2).reshape(1, -1, x.shape[1], x.shape[2])
        wn = w.permute(0, 1, 4, 2, 3).reshape(-1, w.shape[4], w.shape[2], w.shape[3])
        y = F.conv2d(xn, wn, None, stride, pad, groups=B)
        return y.reshape(B, -1, y.shape[2], y.shape[3]).permute(0, 2, 3, 1)
    if w.shape[1] == 1 and w.shape[2] == 1 and stride == 1 and groups == 1:
        return (x.reshape(-1, x.shape[-1]) @ w.reshape(w.shape[0], -1).t()).reshape(*x.shape[:-1], w.shape[0])
    return F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), None, stride, pad, groups=groups).permute(0, 2, 3, 1)


def _epilogue(z, s, b, act, r):
    if s is not None:
        z = z * s
    if b is not None:
        z = z + b
    if r is None:
        return _act64(z, act)
    return _act64(z, act) + r if act & 16 else _act64(z + r, act)


def _magnitude(za, s, b, r):
    a = za if s is None else za * s.abs()
    if b is not None:
        a = a + b.abs()
    return a if r is None else a + r.abs()


def _bounds(A, y64, K, arith, fmt):
    rel, ab = FMT[fmt]
    tail = (C_OUT * U32 + rel) * y64.abs() + ab
    elem = LIP * ((C_ACC * math.sqrt(K) + C_EPI) * U32 + LOLO[arith]) * A + tail
    agg = LIP * ((C_AGG + C_EPI) * U32 + LOLO[arith]) * A + tail
    return elem, agg


class LaunchCheckError(AssertionError):
    pass


class CheckingBackend:
    """ops backend wrapper: every conv / linear launch checked against fp64 of its own operands (see the module docstring)"""

    def __init__(self, inner, label: str = ""):
        self.inner = inner
        self.begin(label)

    def begin(self, label: str):
        """start a new run (a model, a size, a precision): launch indices count from 0 again"""
        self.label, self.index, self.rows, self.failures = label, 0, [], []

    def __getattr__(self, name):
        return getattr(self.inner, name)

    # ---- the wrapped operators --------------------------------------------------------------------------------------------------------------------
    def conv2d(self, x, w, scale, bias, stride, pad, act, residual, out, algo):
        x64, w64, r64 = x.double(), w.double(), _val64(residual)
        geom = self._geom("conv2d", x.shape, w, stride, act, residual, out)
        arith = "fp32" if x.dtype == torch.float32 else "fp16"
        self._launch(geom, arith, [x, w, scale, bias, residual], out, lambda: self.inner.conv2d(x, w, scale, bias, stride, pad, act, residual, out, algo),
                     lambda: self._conv_ref(x64, w64, scale, bias, stride, pad, act, r64))

    def conv2d_pair(self, x, w3, scale, bias, stride, pad, act, residual, out):
        C = x.C
        x64, r64 = _val64(x), _val64(residual)
        w64 = w3[..., :C].double() + w3[..., C:2 * C].double()
        geom = self._geom("conv2d_pair", x.shape, w3, stride, act, residual, out)
        self._launch(geom, "split", [x, w3, scale, bias, residual], out, lambda: self.inner.conv2d_pair(x, w3, scale, bias, stride, pad, act, residual, out),
                     lambda: self._conv_ref(x64, w64, scale, bias, stride, pad, act, r64))

    def stem_conv(self, img, w, scale, bias, mean, std, act, out):
        # the kernel receives mean / std as fp32 and normalises in fp32 (two roundings relative to the normalised value, inside C_EPI)
        m = torch.tensor(mean, dtype=torch.float32).double().to(img.device)
        sd = torch.tensor(std, dtype=torch.float32).double().to(img.device)
        v = img.double() if img.dtype == torch.uint8 else img.double().permute(0, 2, 3, 1)
        x64 = (v - m) / sd
        w64 = w.double()
        geom = self._geom("stem_conv", x64.shape, w, 2, act, None, out)
        self._launch(geom, "fp32", [img, w, scale, bias], out, lambda: self.inner.stem_conv(img, w, scale, bias, mean, std, act, out),
                     lambda: self._conv_ref(x64, w64, scale, bias, 2, 1, act, None))

    def dwconv3x3s2(self, x, w9c, scale, bias, out):
        C = x.shape[-1]
        x64, w64 = x.double(), w9c.double().t().reshape(C, 3, 3, 1)
        geom = self._geom("dwconv3x3s2", x.shape, w64, 2, 0, None, out)
        geom["K"] = 9
        arith = "fp32" if x.dtype == torch.float32 else "fp16"
        self._launch(geom, arith, [x, w9c, scale, bias], out, lambda: self.inner.dwconv3x3s2(x, w9c, scale, bias, out),
                     lambda: self._conv_ref(x64, w64, scale, bias, 2, 1, 0, None, groups=C))

    def linear_rowmax(self, x2d, w, bias, out):
        x64, w64, prev = x2d.double(), w.double(), out.double()
        geom = dict(op="linear_rowmax", M=x2d.shape[0], Cin=x2d.shape[1], Cout=w.shape[0], K=x2d.shape[1], fmt="fp32")
        self._launch(geom, "fp16", [x2d, w, bias], out, lambda: self.inner.linear_rowmax(x2d, w, bias, out), lambda: self._rowmax_ref(x64, w64, bias, prev))

    def linear_rowmax_pair(self, xp, w3, bias, out):
        K = xp.C
        x64, prev = _val64(xp).reshape(-1, K), out.double()
        w64 = w3[:, :K].double() + w3[:, K:2 * K].double()
        geom = dict(op="linear_rowmax_pair", M=x64.shape[0], Cin=K, Cout=w3.shape[0], K=K, fmt="fp32")
        self._launch(geom, "split", [xp, w3, bias], out, lambda: self.inner.linear_rowmax_pair(xp, w3, bias, out), lambda: self._rowmax_ref(x64, w64, bias, prev))

    # ---- references ---------------------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _conv_ref(x64, w64, scale, bias, stride, pad, act, r64, groups=1):
        s = None if scale is None else scale.double()
        b = None if bias is None else bias.double()
        y = _epilogue(_conv64(x64, w64, stride, pad, groups), s, b, act, r64)
        A = _magnitude(_conv64(x64.abs(), w64.abs(), stride, pad, groups), s, b, r64)
        return y, A

    @staticmethod
    def _rowmax_ref(x64, w64, bias, prev):
        """rowmax[m] = max(prev[m], max_n x[m] . w[n] + b[n]); A is the largest magnitude in the row (|max z - max z64| <= max_n |z_n - z64_n|)"""
        b = None if bias is None else bias.double()
        z = x64 @ w64.t()
        za = x64.abs() @ w64.abs().t()
        if b is not None:
            z, za = z + b, za + b.abs()
        return torch.maximum(prev, z.max(-1).values), za.max(-1).values

    # ---- the launch and its checks -------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _geom(op, xshape, w, stride, act, residual, out):
        B, H, W, Cin = xshape
        Cout, KH, KW = w.shape[-4], w.shape[-3], w.shape[-2]
        o = out.hi if isinstance(out, Pair) else out
        fmt = "pair" if isinstance(out, Pair) else ("fp32" if out.dtype == torch.float32 else "fp16")
        Ho, Wo = o.shape[1], o.shape[2]
        pitch = o.stride(-2)
        return dict(op=op, fmt=fmt, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=KH, stride=stride, K=KH * KW * Cin, act=act & 15,
                    res=None if residual is None else ("post" if act & 16 else "pre"), per_image=w.dim() == 5,
                    out_slice=(Cout < (out.Ctot if isinstance(out, Pair) else pitch)), flat_linear=(KH == 1 and B == 1 and H == 1 and op != "stem_conv"),
                    batch_strided=bool(B > 1 and o.stride(0) != Ho * Wo * pitch), odd_map=bool(H % 2 or W % 2), Ho=Ho, Wo=Wo)

    def _launch(self, geom, arith, inputs, out, call, ref):
        idx = self.index
        self.index += 1
        geom = dict(geom, arith=arith, site=_site())
        ovs = _views(out)
        # snapshots: the inputs (bit patterns) and the output's storage span
        ins = [(v, v.clone()) for t in inputs for v in _views(t)]
        first = min(_extent(v)[0] for v in ovs)
        last = max(_extent(v)[1] for v in ovs)
        pitch = ovs[0].stride(-2) if ovs[0].dim() >= 2 else 1
        flat = _flat(ovs[0])
        a, b = max(0, first - pitch), min(flat.numel(), last + pitch + 1)
        span0 = flat[a:b].clone()
        inside = torch.zeros(b - a, dtype=torch.bool, device=flat.device)
        for v in ovs:
            inside.as_strided(v.shape, v.stride(), v.storage_offset() - a).fill_(True)
        call()
        if flat.is_cuda:
            torch.cuda.synchronize()
        y64, A = ref()
        y = _val64(out)
        fails = []
        # 1 / 2: per element and per launch
        elem, agg = _bounds(A, y64, geom["K"], arith, geom["fmt"])
        err = (y - y64).abs()
        bad = ~(err <= elem)  # NaN counts as a failure
        ratio = torch.where(err == 0, torch.zeros_like(err), err / elem)
        ratio = torch.where(torch.isnan(ratio), torch.full_like(err, float("inf")), ratio)
        worst = int(ratio.reshape(-1).argmax()) if ratio.numel() else 0
        elem_ratio = float(ratio.reshape(-1)[worst]) if ratio.numel() else 0.0
        en, an, bn = float(torch.linalg.vector_norm(err)), float(torch.linalg.vector_norm(A)), float(torch.linalg.vector_norm(agg))
        agg_ratio = en / bn if bn > 0 else (0.0 if en == 0 else float("inf"))
        if math.isnan(agg_ratio):
            agg_ratio = float("inf")
        if bool(bad.any()):
            at = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), tuple(y.shape)))
            fails.append(f"element {at}: y={float(y.reshape(-1)[worst]):.9g} ref={float(y64.reshape(-1)[worst]):.9g} err={float(err.reshape(-1)[worst]):.3e} "
                         f"bound={float(elem.reshape(-1)[worst]):.3e} ({int(bad.sum())} of {bad.numel()} elements over)")
        if not agg_ratio <= 1.0:
            fails.append(f"aggregate ||y - y64|| = {en:.3e} over ||agg bound|| = {bn:.3e} (||A|| = {an:.3e})")
        # 3: a Pair output encodes its value
        if isinstance(out, Pair):
            hi, lo = out.hi, out.lo
            toward = torch.where(lo >= 0, torch.full_like(hi, float("inf")), torch.full_like(hi, float("-inf")))
            gap = (torch.nextafter(hi, toward).float() - hi.float()).abs()
            enc = torch.isfinite(hi) & (2 * lo.float().abs() <= gap)
            if not bool(enc.all()):
                at = tuple(int(i) for i in (~enc).nonzero()[0])
                fails.append(f"pair encoding at {at}: hi={float(hi[at]):.9g} lo={float(lo[at]):.9g} is not a nearest fp16 of hi + lo ({int((~enc).sum())} elements)")
        # 4: nothing outside the output view in its span changed
        moved = (_bits(flat[a:b]) != _bits(span0)) & ~inside
        if bool(moved.any()):
            off = a + int(moved.nonzero()[0])
            fails.append(f"wrote outside the output view: storage element {off} (view elements {first}..{last}, pitch {pitch}; {int(moved.sum())} elements changed)")
        # 5: the inputs are unchanged (an input sharing the output's storage is left to check 4)
        for v, v0 in ins:
            if v.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr():
                continue
            if not torch.equal(_bits(v), _bits(v0)):
                fails.append(f"an input of shape {tuple(v.shape)} changed")
        row = dict(geom, label=self.label, index=idx, elem_ratio=elem_ratio, agg_ratio=agg_ratio, agg_rel_u32=(en / an / U32) if an > 0 else 0.0, ok=not fails)
        self.rows.append(row)
        for f in fails:
            self.failures.append(f"{self.label} launch #{idx} {_describe(geom)}: {f}")

    def raise_failures(self, limit: int = 12):
        if self.failures:
            more = f"\n... and {len(self.failures) - limit} more" if len(self.failures) > limit else ""
            raise LaunchCheckError(f"{len(self.failures)} check(s) failed:\n" + "\n".join(self.failures[:limit]) + more)


def _describe(g):
    if g["op"].startswith("linear_rowmax"):
        return f"{g['op']} [{g['arith']}] M={g['M']} K={g['K']} N={g['Cout']} at {g['site']}"
    return (f"{g['op']} [{g['arith']} -> {g['fmt']}] {g['B']}x{g['H']}x{g['W']}x{g['Cin']} -> {g['Ho']}x{g['Wo']}x{g['Cout']} k{g['k']} s{g['stride']} "
            f"act {g['act']}{'' if g['res'] is None else ' res ' + g['res']}{' per-image' if g['per_image'] else ''}{' slice' if g['out_slice'] else ''}"
            f"{' batch-strided' if g['batch_strided'] else ''} at {g['site']}")


def seeded_model(name: str, precision: str, device: str = "cpu"):
    """the registry model `name` with the seeded weights of its manifest (fai-detr-l-coco, which has none, seeds its own state_dict the same way)"""
    from focoos_b200 import ModelManager
    from focoos_b200.utils.seeded_weights import seeded_state_dict
    from tests.parity_utils import GOLDEN, manifest_template

    m = ModelManager.get(name, precision=precision).model
    man = name.replace("-", "_")
    template = manifest_template(man) if os.path.exists(os.path.join(GOLDEN, f"{man}_state_dict_manifest.json")) else m.state_dict()
    m.load_state_dict(seeded_state_dict(template, 0), strict=True)
    return m.cuda() if device == "cuda" else m


def synth_batch(seed: int, B: int, H: int, W: int, device: str = "cpu"):
    """B synthetic images [B,3,H,W] fp32 0..255"""
    from oracle.gen_golden import synth_images

    return torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in synth_images(seed, [(H, W)] * B)]).to(device)


def summarize(rows):
    """{arith: (worst per-element ratio, its launch, worst aggregate ratio, its launch)} over report rows"""
    out = {}
    for r in rows:
        cur = out.setdefault(r["arith"], [0.0, None, 0.0, None])
        if r["elem_ratio"] >= cur[0]:
            cur[0], cur[1] = r["elem_ratio"], f"{r['label']} #{r['index']} {_describe(r)}"
        if r["agg_ratio"] >= cur[2]:
            cur[2], cur[3] = r["agg_ratio"], f"{r['label']} #{r['index']} {_describe(r)}"
    return out
