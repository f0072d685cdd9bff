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

The backward operators of the fine-tune step are wrapped the same way: conv_wgrad, conv_wgrad_tc, conv_wgrad_tc_f16, dilate2, colsum and add_act.  Before
each of these launches the output is filled with NaN, so an element the kernel never writes, or a kernel that adds onto `dw` although the call passes
accumulate = 0, fails check 1.
  * weight gradient  dW[co,kh,kw,ci] = sum over the K = B*Ho*Wo output pixels of dy * x, against fp64 of the operand values the launch received (the
    fp32 tensors; hi + lo of both [hi | lo] pairs; the fp16 values of the amp operands).  A = the same sum over |x| * |dy|.  The split products omit
    lo x dy_lo (LOLO); the fp16 products are exact in fp32, so only the accumulation term remains.  With K up to 1.6 M (the 32-channel convs of the
    stem at bs=16, 640x640) the per-element bar is C_ACC * sqrt(K) * u32 ~ 3e-4 of A, far above a dropped hi x dy_lo product (each term 2^-11 of its
    product).  The per-launch bar (C_AGG + LOLO) ~ 16 u32 of ||A|| is what sees it: the dropped terms carry the rounding residual of dy, whose sign is
    unrelated to the product's, so they add up as a random walk to ~2^-12 * sqrt(K) * rms(dy x) per element - above 16 u32 * A ~ 16 u32 * K * mean|dy x|
    while K stays below ~10^5 (every launch of a small step; at bs=16 the weight gradients of the deep stages, not the 1.6 M-pixel stem convs).
  * dilate2          exact: dy at the even (h, w), zeros elsewhere.
  * colsum           fp32 sum of K = R rows: A = the column sum of |x|.
  * add_act          forward act(a + b), or the gradient dy * act'(a + b).  a + b is one fp32 rounding and exact in fp64, so the forward sum (no
                     activation) and ReLU equal fp32(a + b) exactly, and the pass-through gradient and the ReLU gradient gate (the sign of the
                     rounded sum is the sign of the exact one) equal dy exactly.  The smooth activations (u = u32, z = a + b):
      forward        the rounding of z moves the result by at most LIP * u * |z|; GELU = z/2 * (1 + erf(z / sqrt 2)) adds erff's 2 ulp (<= 2u, the values
                     are below 1) and the two roundings of its argument (slope of erf times 2u|t| <= 1u) to 1 + erf, i.e. <= 1.5 u |z| after the
                     product with z/2, and two roundings of the result; SiLU = z / (1 + expf(-z)) has expf's 2 ulp, the sum and the quotient, all
                     relative to the result (<= 6 u |y|, and |y| <= |z|):  bound = (LIP + C_OUT) * u * |z| + C_OUT * u * |y64|
      GELU gradient  act' = Phi(z) + z phi(z): Phi through erff as above (<= 2u), z phi(z) <= 0.25 with expf's 2 ulp, the argument -z^2/2 (relative
                     z^2 u, <= 0.5u absolute after the factor z phi(z)) and two products (<= 2u); the rounding of z (|z act''(z)| <= 0.4, 0.4u); the sum
                     (1.13u): <= 6u in all, so  bound = 2 * C_OUT * u * |dy| + C_OUT * u * |g64|
      SiLU gradient  act' = s (1 + z (1 - s)), s = 1 / (1 + expf(-z)) rounded to <= 2u absolute, which 1 - s carries unchanged and z multiplies:
                     bound = 2 * C_OUT * u * (1 + |z|) * |dy| + C_OUT * u * |g64|
    An element-wise launch has no accumulation to average over, so its per-launch bar is the norm of the per-element bar.
"Exact" compares values: +0 and -0 are equal (a ReLU gradient dy * 0 is -0 for a negative dy).
"""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.nn.functional as F

from focoos_b200 import ops
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
# tensor-core products of fp16 operands (split and fp16 arithmetic) have an absolute floor: a product of two fp16 values is a multiple of 2^-48, and the
# wgmma sums lose products near that scale.  Measured on the fine-tune step's linear data gradients (K = 256, outputs ~1e-8 where dy lies at the fp16
# underflow): errors up to 2^-40.4 against fp64 of the same fp16 operands, in elements whose bar without this term was 2^-42.  Per element: K * 2^-48
# (1e-12 at K = 256), nothing next to the bars of outputs of ordinary magnitude.
TC_ABS = {"split": 2.0 ** -48, "fp16": 2.0 ** -48}


_TORCH_DIR = os.path.dirname(torch.__file__) + os.sep


def _site():
    """file:function:line of the model code that made the launch: the first frame outside the operator layer, this module, the autograd functions
    (autograd_ops.py), torch itself and the engines' generic layer calls (_conv / _linear).  A backward launch is made by the autograd engine, not by the
    model, so it is named by the autograd function's backward line (autograd_ops.py:Conv2dFn.backward:137)."""
    f = sys._getframe(2)
    skip = (os.sep + "ops.py", os.sep + "conv_launch_check.py", os.sep + "autograd_ops.py")
    while f is not None:
        fn = f.f_code.co_filename
        if fn.endswith(os.sep + "autograd_ops.py") and f.f_code.co_name == "backward":
            return f"autograd_ops.py:{f.f_code.co_qualname}:{f.f_lineno}"
        if not (fn.endswith(skip) or fn.startswith(_TORCH_DIR) or f.f_code.co_name in ("_conv", "_linear")):
            break
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


def _bounds(A, y64, K, arith, fmt, lip=LIP):
    rel, ab = FMT[fmt]
    tail = (C_OUT * U32 + rel) * y64.abs() + ab
    elem = lip * ((C_ACC * math.sqrt(K) + C_EPI) * U32 + LOLO[arith]) * A + tail + K * TC_ABS.get(arith, 0.0)
    agg = lip * ((C_AGG + C_EPI) * U32 + LOLO[arith]) * A + tail
    return elem, agg


def _wgrad64(x64, dy64, KH, KW, stride, pad):
    """fp64 weight gradient [Cout,KH,KW,Cin] of an NHWC conv: one GEMM dy^T @ x per filter tap, over the tap's shifted (and, for stride 2,
    element-strided) view of the zero-padded input"""
    B, Ho, Wo, Cout = dy64.shape
    Cin = x64.shape[-1]
    d = dy64.reshape(-1, Cout).t()
    if KH == 1 and KW == 1 and stride == 1 and pad == 0:
        return (d @ x64.reshape(-1, Cin)).reshape(Cout, 1, 1, Cin)
    xp = F.pad(x64, (0, 0, pad, pad, pad, pad))
    dw = torch.empty((Cout, KH, KW, Cin), dtype=torch.float64, device=x64.device)
    for kh in range(KH):
        for kw in range(KW):
            xs = xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride, :]
            dw[:, kh, kw, :] = d @ xs.reshape(-1, Cin)
    return dw


def _pair64(t, C):
    """fp64 values of a dense [hi | lo] fp16 pair tensor [..., 2C]"""
    return t[..., :C].double() + t[..., C:2 * C].double()


def _stem_wgrad(x_shape, Cout, KH, stride, pad):
    """fb200_conv_wgrad runs the stem's weight gradient (3x3 stride 2, at most 4 input channels, 32 outputs) on its dedicated kernel.  This is the
    dispatch condition of fb200_conv_wgrad (csrc/bwd_conv_norm.cu) and must change with it; its other clause, that the workspace holds one partial per
    block, always holds: fb200_conv_wgrad_workspace_bytes sizes the workspace for 2 * kNumSMs partials."""
    return KH == 3 and stride == 2 and pad == 1 and x_shape[-1] <= 4 and Cout == 32


class LaunchCheckError(AssertionError):
    pass


class CheckingBackend:
    """ops backend wrapper: every conv / linear launch checked against fp64 of its own operands (see the module docstring)"""

    def __init__(self, inner, label: str = "", mode: str = ""):
        self.inner = inner
        self.begin(label, mode)

    def begin(self, label: str, mode: str = ""):
        """start a new run (a model, a size, a precision): launch indices count from 0 again; `mode` (a training arithmetic) is copied into every row"""
        self.label, self.mode, self.index, self.rows, self.failures = label, mode, 0, [], []

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

    # ---- the backward operators of the fine-tune step ----------------------------------------------------------------------------------------------
    def conv_wgrad(self, x, dy, KH, KW, stride, pad, dw):
        x64, dy64 = x.double(), dy.double()
        geom = self._wgrad_geom("conv_wgrad", x.shape, dy.shape, KH, stride, "stem" if _stem_wgrad(x.shape, dy.shape[-1], KH, stride, pad) else "simt")
        self._launch(geom, "fp32", [x, dy], dw, self._filled(dw, lambda: self.inner.conv_wgrad(x, dy, KH, KW, stride, pad, dw)),
                     lambda: self._wgrad_ref(x64, dy64, KH, KW, stride, pad, "fp32"))

    def conv_wgrad_tc(self, x_pair, dy_pair, KH, KW, stride, pad, dw):
        Cin, Cout = x_pair.shape[-1] // 2, dy_pair.shape[-1] // 2
        x64, dy64 = _pair64(x_pair, Cin), _pair64(dy_pair, Cout)
        geom = self._wgrad_geom("conv_wgrad_tc", x64.shape, dy64.shape, KH, stride, "split")
        self._launch(geom, "split", [x_pair, dy_pair], dw, self._filled(dw, lambda: self.inner.conv_wgrad_tc(x_pair, dy_pair, KH, KW, stride, pad, dw)),
                     lambda: self._wgrad_ref(x64, dy64, KH, KW, stride, pad, "split"))

    def conv_wgrad_tc_f16(self, x16, dy16, KH, KW, stride, pad, dw):
        x64, dy64 = x16.double(), dy16.double()
        geom = self._wgrad_geom("conv_wgrad_tc_f16", x16.shape, dy16.shape, KH, stride, "f16")
        self._launch(geom, "fp16", [x16, dy16], dw, self._filled(dw, lambda: self.inner.conv_wgrad_tc_f16(x16, dy16, KH, KW, stride, pad, dw)),
                     lambda: self._wgrad_ref(x64, dy64, KH, KW, stride, pad, "fp16"))

    def dilate2(self, dy, out):
        dy64 = dy.double()
        B, Ho, Wo, C = dy.shape
        geom = dict(op="dilate2", fmt="fp32", B=B, H=Ho, W=Wo, Cin=C, Cout=C, Ho=out.shape[1], Wo=out.shape[2], K=1, odd_map=bool(out.shape[1] % 2 or out.shape[2] % 2))

        def ref():
            y = torch.zeros(out.shape, dtype=torch.float64, device=out.device)
            y[:, 0:2 * Ho:2, 0:2 * Wo:2] = dy64
            return y, torch.zeros_like(y), torch.zeros_like(y)
        self._launch(geom, "exact", [dy], out, self._filled(out, lambda: self.inner.dilate2(dy, out)), ref)

    def colsum(self, x2d, out):
        x64 = x2d.double()
        geom = dict(op="colsum", fmt="fp32", M=x2d.shape[0], Cout=x2d.shape[1], K=x2d.shape[0])

        def ref():
            y, A = x64.sum(0), x64.abs().sum(0)
            return (y, *_bounds(A, y, x64.shape[0], "fp32", "fp32", lip=1.0), A)
        self._launch(geom, "fp32", [x2d], out, self._filled(out, lambda: self.inner.colsum(x2d, out)), ref)

    def add_act(self, a, b, dy, act, out):
        z64 = a.double() if b is None else a.double() + b.double()
        dy64 = None if dy is None else dy.double()
        geom = dict(op="add_act", fmt="fp32", act=act, grad=dy is not None, M=a.numel(), Cout=a.shape[-1], K=1, sum=b is not None)
        exact = act in (ops.ACT_NONE, ops.ACT_RELU)
        self._launch(geom, "exact" if exact else "fp32", [a, b, dy], out, self._filled(out, lambda: self.inner.add_act(a, b, dy, act, out)),
                     lambda: self._add_act_ref(z64, dy64, act))

    # ---- references ---------------------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _wgrad_ref(x64, dy64, KH, KW, stride, pad, arith):
        y = _wgrad64(x64, dy64, KH, KW, stride, pad)
        A = _wgrad64(x64.abs(), dy64.abs(), KH, KW, stride, pad)
        return (y, *_bounds(A, y, dy64.shape[0] * dy64.shape[1] * dy64.shape[2], arith, "fp32", lip=1.0), A)

    @staticmethod
    def _add_act_ref(z, dy, act):
        """the result and its bounds (module docstring): exact for no activation and ReLU, unit-roundoff bounds for SiLU and GELU"""
        if dy is None:
            if act in (ops.ACT_NONE, ops.ACT_RELU):  # the correctly rounded fp32 sum (fp64 holds a + b exactly, so rounding it once more is that)
                y = _act64(z.float().double(), act)
                return y, torch.zeros_like(y), torch.zeros_like(y)
            y = _act64(z, act)
            elem = (LIP + C_OUT) * U32 * z.abs() + C_OUT * U32 * y.abs()
            return y, elem, elem
        if act == ops.ACT_NONE:
            return dy.clone(), torch.zeros_like(dy), torch.zeros_like(dy)
        if act == ops.ACT_RELU:
            return dy * (z > 0).double(), torch.zeros_like(dy), torch.zeros_like(dy)
        if act == ops.ACT_SILU:
            s = torch.sigmoid(z)
            g = dy * s * (1.0 + z * (1.0 - s))
            elem = 2 * C_OUT * U32 * (1.0 + z.abs()) * dy.abs() + C_OUT * U32 * g.abs()
        else:
            assert act == ops.ACT_GELU, f"unknown activation {act}"
            g = dy * (0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi))
            elem = 2 * C_OUT * U32 * dy.abs() + C_OUT * U32 * g.abs()
        return g, elem, elem

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
    def _filled(out, call):
        """the launch, with its fp32 output filled with the NaN sentinel first (an element left unwritten, or added onto, stays NaN)"""
        def run():
            out.fill_(float("nan"))
            call()
        return run

    @staticmethod
    def _wgrad_geom(op, xshape, dyshape, k, stride, kernel):
        B, H, W, Cin = xshape
        _, Ho, Wo, Cout = dyshape
        return dict(op=op, fmt="fp32", kernel=kernel, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, stride=stride, K=B * Ho * Wo, Ho=Ho, Wo=Wo,
                    odd_map=bool(H % 2 or W % 2), linear=(k == 1 and B == 1 and H == 1))

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
        r = ref()  # (y64, A), or (y64, per-element bound, per-launch bound[, A]) for an operator with bounds of its own
        y64, (elem, agg) = r[0], (r[1:3] if len(r) >= 3 else _bounds(r[1], r[0], geom["K"], arith, geom["fmt"]))
        A = r[1] if len(r) == 2 else (r[3] if len(r) == 4 else None)
        y = _val64(out)
        fails = []
        # 1 / 2: per element and per launch
        err = (y - y64).abs()
        bad = ~(err <= elem)  # NaN counts as a failure
        ratio = torch.where(err == 0, torch.zeros_like(err), err / elem)
        ratio = torch.where(torch.isnan(ratio), torch.full_like(err, float("inf")), ratio)
        worst = int(ratio.reshape(-1).argmax()) if ratio.numel() else 0
        elem_ratio = float(ratio.reshape(-1)[worst]) if ratio.numel() else 0.0
        en, bn = float(torch.linalg.vector_norm(err)), float(torch.linalg.vector_norm(agg))
        an = float(torch.linalg.vector_norm(A)) if A is not None else 0.0
        agg_ratio = en / bn if bn > 0 else (0.0 if en == 0 else float("inf"))
        if math.isnan(agg_ratio):
            agg_ratio = float("inf")
        if bool(bad.any()):
            at = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), tuple(y.shape)))
            fails.append(f"element {at}: y={float(y.reshape(-1)[worst]):.9g} ref={float(y64.reshape(-1)[worst]):.9g} err={float(err.reshape(-1)[worst]):.3e} "
                         f"bound={float(elem.reshape(-1)[worst]):.3e} ({int(bad.sum())} of {bad.numel()} elements over)")
        if not agg_ratio <= 1.0:
            fails.append(f"aggregate ||y - y64|| = {en:.3e} over ||agg bound|| = {bn:.3e}" + (f" (||A|| = {an:.3e})" if A is not None else ""))
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
        row = dict(geom, label=self.label, mode=self.mode, index=idx, elem_ratio=elem_ratio, agg_ratio=agg_ratio, agg_rel_u32=(en / an / U32) if an > 0 else 0.0, ok=not fails)
        self.rows.append(row)
        for f in fails:
            self.failures.append(f"{self.label} launch #{idx} {_describe(geom)}: {f}")

    def raise_failures(self, limit: int = 12):
        if self.failures:
            more = f"\n... and {len(self.failures) - limit} more" if len(self.failures) > limit else ""
            raise LaunchCheckError(f"{len(self.failures)} check(s) failed:\n" + "\n".join(self.failures[:limit]) + more)


def _describe(g):
    if g["op"].startswith("conv_wgrad"):
        return (f"{g['op']} [{g['arith']}, {g['kernel']}] x {g['B']}x{g['H']}x{g['W']}x{g['Cin']} dy {g['Ho']}x{g['Wo']}x{g['Cout']} k{g['k']} s{g['stride']} "
                f"K={g['K']} at {g['site']}")
    if g["op"] == "dilate2":
        return f"dilate2 {g['B']}x{g['H']}x{g['W']}x{g['Cin']} -> {g['Ho']}x{g['Wo']} at {g['site']}"
    if g["op"] == "colsum":
        return f"colsum [{g['arith']}] R={g['M']} C={g['Cout']} at {g['site']}"
    if g["op"] == "add_act":
        return f"add_act act {g['act']}{' gradient' if g['grad'] else ''}{' of a + b' if g['sum'] else ''} n={g['M']} at {g['site']}"
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


TRAIN_MODEL = "fai-detr-l-coco"


def train_model(mode: str, device: str = "cpu"):
    """fai-detr-l-coco with its seeded weights, classifiers desaturated as in the training goldens, in train mode with the training arithmetic `mode`
    ("fp32", "fp32_tc" or "amp": the fp32_tc model with TrainerArgs.amp_enabled)"""
    from focoos_b200.utils.seeded_weights import desaturate_classifiers

    m = seeded_model(TRAIN_MODEL, "fp32" if mode == "fp32" else "fp32_tc", device)
    m.load_state_dict(desaturate_classifiers(m.state_dict()), strict=True)
    if mode == "amp":
        m.train_precision = "amp"
    m.train()
    assert m.train_graph().prec == mode
    return m


def train_step(m, B: int, H: int, W: int, device: str = "cpu"):
    """one TrainStep (forward, criterion, loss-scaled backward, clipped AdamW) on synthetic images and targets; returns the losses"""
    from focoos_b200.criterion import DETRTargets
    from focoos_b200.train_step import FlatAdamW, TrainStep, get_optimizer_params
    from oracle.gen_golden_train import synth_targets

    opt = FlatAdamW(get_optimizer_params(m, base_lr=1e-4, weight_decay=1e-4, weight_decay_norm=0.0, backbone_multiplier=0.1), clip_gradients=0.1, amp=True)
    x = synth_batch(5, B, H, W, device)
    targets = [DETRTargets(labels=t[0].to(device), boxes=t[1].to(device)) for t in synth_targets(6, B, m.config.num_classes)]
    return TrainStep(m, opt)(x, targets)
