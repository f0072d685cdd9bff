"""Multi-head attention (head_dim 32) forward and backward against a float64 reference written in this file.

Entry points and the kernels they reach:
- `fb200_attention`: `attention_kernel<float>`, `attention_kernel<__half>` (fp16 rows that are not 16-byte aligned), `attention_mma_kernel` (fp16
  tensor cores); above the shared-memory ceilings of these resident kernels, the streaming kernels of `fb200_attention_masked` without a mask.
- `fb200_attention_split`: `attention_mma_split_kernel` (fp32 or [hi | lo] pair output); above its ceiling fp32 rows are streamed by
  `attention_mma_split_stream_kernel<false>`.
- `fb200_attention_masked`: `attention_mma_stream_kernel` (fp16, aligned), `attention_masked_kernel<float / __half>`.
- `fb200_attention_masked_split`: `attention_mma_split_stream_kernel<false>` (fp32 K/V) and `<true>` (pair K/V).
- `fb200_attention_bwd`: `attention_bwd_kernel<36>` / `<33>`.

Rows.  Every (query, head) row has a kind: unit-scale random, peaked (one key >= 30 above every other, in the first 64-key block or in the last
one), huge-logit (scaled scores spanning +-80), rising (the row maximum rises with every key, so every 64-key block rescales), uniform (q = 0).
Masked cases add mask rows with no allowed key, exactly one allowed key (at 0, Lk-1 and on both sides of the 64 / 128 / 256-key boundaries),
masked leading blocks, alternating masks and no mask at all.

Bars, as a per-element bound on |got - want|:
- FWD_TOL = 2e-5 of the output scale (max |want|) for every fp32 and split path;
- fp16 outputs also one fp16 rounding of the output and the fp16 rounding of P in the P.V product: 2^-11 * (|want| + P.|V|);
- GRAD_TOL = 5e-5 of each gradient's own scale;
- on the peaked, huge-logit and rising rows (q far from unit scale) the first-order effect of rounding the scores, derived at `score_terms`.

`-k self_check` runs without a GPU: it checks the reference and the bounds before any GPU test relies on them."""
import math
import re
import time

import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import autograd_ops as A
from focoos_b200 import ops
from oracle.ops_ref import RefBackend

pytestmark = pytest.mark.timeout(900)
gpu = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
HD = 32
SCALE = 1 / math.sqrt(HD)
U = 2.0 ** -24   # fp32 unit roundoff
FWD_TOL = 2e-5
GRAD_TOL = 5e-5
NAN = float("nan")

KINDS = ("random", "peak_first", "peak_last", "huge", "rising", "uniform")
KIND_P = [0.4, 0.1, 0.1, 0.15, 0.15, 0.1]
FLAGGED = (1, 2, 3, 4)   # rows whose q is far from unit scale: their bound carries the score-rounding term
PEAK_GAP, HUGE_SPAN, RISE_SPAN = 32.0, 80.0, 16.0


# ---- float64 reference --------------------------------------------------------------------------------------------------------------------------------------
def _split_heads(t, heads):
    """[B, L, heads*32] -> [B, heads, L, 32] in float64"""
    B, L, _ = t.shape
    return t.to(F64).reshape(B, L, heads, HD).transpose(1, 2)


def _merge_heads(t):
    B, h, L, d = t.shape
    return t.transpose(1, 2).reshape(B, L, h * d)


def dead_keys(mask, Lk):
    """[B, Lq, Lk] bool, the keys a query does not attend to (fai_mf/modelling.py:505-513): mask byte != 0, except in a row where every key is
    masked, which attends everywhere.  Bytes past Lk (the row padding) are not keys."""
    dead = mask[:, :, :Lk] != 0
    return dead & ~dead.all(-1, keepdim=True)


def probs64(q, k, heads, scale, mask=None):
    """softmax(q k^T * scale) per head, [B, heads, Lq, Lk] float64; masked keys get -inf"""
    s = _split_heads(q, heads) @ _split_heads(k, heads).transpose(-1, -2) * scale
    if mask is not None:
        s = s.masked_fill(dead_keys(mask, k.shape[1])[:, None], float("-inf"))
    return torch.softmax(s, -1)


def attn64(q, k, v, heads, scale, mask=None):
    """q [B, Lq, C], k / v [B, Lk, C] -> [B, Lq, C] float64"""
    return _merge_heads(probs64(q, k, heads, scale, mask) @ _split_heads(v, heads))


def attn_bwd64(q, k, v, dout, heads, scale):
    """(dq, dk, dv) of attn64, written out: dV = P^T dO, dP = dO V^T, dS = P * (dP - rowsum(P * dP)) * scale, dQ = dS K, dK = dS^T Q"""
    P = probs64(q, k, heads, scale)
    Q, K, V, dO = (_split_heads(t, heads) for t in (q, k, v, dout))
    dP = dO @ V.transpose(-1, -2)
    dS = P * (dP - (P * dP).sum(-1, keepdim=True)) * scale
    return _merge_heads(dS @ K), _merge_heads(dS.transpose(-1, -2) @ Q), _merge_heads(P.transpose(-1, -2) @ dO)


# ---- bounds ----------------------------------------------------------------------------------------------------------------------------------------------------
def score_terms(q, k, v, heads, scale, kind, mask=None):
    """First-order effect of rounding the scores, on the flagged rows (zero on the others).

    A dot product of D = 32 fp32 products is off by at most D*u*sum_d |q_d||k_d| (u = 2^-24, first order; the split kernels drop the lo*lo products,
    2^-22 each, which is inside the same bound), so the scaled score s_j of key j is off by d_j <= D*u*scale*a_j, a_j = sum_d |q_d||k_jd|.  The row
    maximum, the exponent and the normalisation only ever see these scores, so the probabilities move by dp_j = p_j (d_j - dbar), dbar = sum_j p_j d_j,
    and the output o = sum_j p_j v_j by sum_j p_j (d_j - dbar) (v_j - o) (the dbar * o terms cancel).  o is a convex combination of the v_j, so per
    column |v_j - o| <= range(v) = max_j v_j - min_j v_j and
        |do| <= 2 * D*u*scale * (sum_j p_j a_j) * range(v).
    Returns (the bound [B, heads, Lq, 32], the relative bound of each probability r_ij = D*u*scale*(a_ij + sum_j p_ij a_ij) [B, heads, Lq, Lk], P)."""
    P = probs64(q, k, heads, scale, mask)
    Q, K, V = (_split_heads(t, heads) for t in (q, k, v))
    a = Q.abs() @ K.abs().transpose(-1, -2)
    pa = (P * a).sum(-1, keepdim=True)
    flag = torch.isin(kind, torch.tensor(FLAGGED, device=kind.device)).transpose(1, 2)[..., None].to(F64)   # [B, heads, Lq, 1]
    rng = (V.amax(2) - V.amin(2))[:, :, None, :]
    return 2 * HD * U * scale * pa * rng * flag, HD * U * scale * (a + pa) * flag, P


def out_bound(q, k, v, heads, scale, kind, mask=None, f16=False):
    """(want [B, Lq, C], per-element bound of |got - want|) for a forward output"""
    term, _, P = score_terms(q, k, v, heads, scale, kind, mask)
    V = _split_heads(v, heads)
    want = P @ V
    bound = FWD_TOL * float(want.abs().max()) + term
    if f16:   # one rounding of the output, and P rounded to fp16 before the P.V product (the normalisation uses the unrounded P)
        bound = bound + 2.0 ** -11 * (want.abs() + P @ V.abs())
    return _merge_heads(want), _merge_heads(bound)


def grad_bounds(q, k, v, o, dout, heads, scale, kind):
    """((dq, dk, dv) fp64, their per-element bounds).  Every gradient gets GRAD_TOL of its own scale.  On the flagged rows the kernel recomputes
    p_ij with a relative error up to r_ij (score_terms), and D_i = rowsum(dO_i * o_i) takes the forward error of o_i (o is the kernel's output):
        dv_j  gets sum_i p_ij r_ij |dO_i|,
        ds_ij = scale * p_ij (dp_ij - D_i) gets scale * G_ij, G_ij = p_ij (r_ij |dp_ij - D_i| + sum_c |dO_ic| do_ic),
        dq_i = sum_j ds_ij k_j and dk_j = sum_i ds_ij q_i get scale * G |K| and scale * G^T |Q|."""
    grads = attn_bwd64(q, k, v, dout, heads, scale)
    term, r, P = score_terms(q, k, v, heads, scale, kind)
    Q, K, V, dO = (_split_heads(t, heads) for t in (q, k, v, dout))
    dP = dO @ V.transpose(-1, -2)
    Dr = (P * dP).sum(-1, keepdim=True)
    G = P * (r * (dP - Dr).abs() + (dO.abs() * term).sum(-1, keepdim=True))
    extra = (scale * G @ K.abs(), scale * G.transpose(-1, -2) @ Q.abs(), (P * r).transpose(-1, -2) @ dO.abs())
    return grads, tuple(GRAD_TOL * float(g.abs().max()) + _merge_heads(e) for g, e in zip(grads, extra))


def assert_within(got, want, bound, what):
    got = got.detach().to(want.device, F64)
    err = (got - want).abs()
    bad = ~(err <= bound)   # NaN counts as off
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off; first at flat index {i}: got {float(got.flatten()[i]):.6e}, "
                             f"want {float(want.flatten()[i]):.6e}, bound {float(torch.as_tensor(bound).expand_as(err).flatten()[i]):.3e}; "
                             f"max|d| = {float(err.nan_to_num(float('inf')).max()):.3e}, scale {float(want.abs().max()):.3e}")


# ---- inputs --------------------------------------------------------------------------------------------------------------------------------------------------------
def make_qkv(B, Lq, Lk, heads, seed, dtype=torch.float32):
    """(q [B, Lq, C], k, v [B, Lk, C] in `dtype`, kind [B, Lq, heads] int64: index into KINDS).

    Keys: unit normal, except that their component along one unit direction u_h per head ramps from 0 to 4 with the key index; a rising row
    is q_h = beta * u_h, whose scores then grow with every key (scaled from 0 to RISE_SPAN).  A peaked row is q_h = c * k_j*/|k_j*| with j* drawn
    in the first 64-key block or in the last block and c set so that the scaled score of j* is PEAK_GAP above every other key (rows whose j*
    would need more than a 64-fold q fall back to random).  A huge-logit row is a random q scaled until its largest |scaled score| is HUGE_SPAN."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((B, Lq, heads, HD), generator=g, dtype=F64)
    k = torch.randn((B, Lk, heads, HD), generator=g, dtype=F64)
    v = torch.randn((B, Lk, heads, HD), generator=g, dtype=F64)
    kind = torch.multinomial(torch.tensor(KIND_P), B * Lq * heads, replacement=True, generator=g).view(B, Lq, heads)
    u = F.normalize(torch.randn((heads, HD), generator=g, dtype=F64), dim=-1)
    ramp = 4.0 * torch.arange(Lk, dtype=F64) / Lk
    k = k - (k * u).sum(-1, keepdim=True) * u + ramp.view(1, Lk, 1, 1) * u
    k = k.to(dtype).to(F64)   # the scores below are those of the rounded keys
    # peaked
    last0 = (Lk - 1) // 64 * 64
    first = torch.randint(0, min(64, Lk), (B, Lq, heads), generator=g)
    last = last0 + torch.randint(0, Lk - last0, (B, Lq, heads), generator=g)
    jstar = torch.where(kind == 2, last, first)
    bi, hi = torch.arange(B).view(B, 1, 1), torch.arange(heads).view(1, 1, heads)
    ks = k[bi, jstar, hi]
    us = F.normalize(ks, dim=-1)
    proj = torch.einsum("bqhd,bkhd->bqhk", us, k)
    proj.scatter_(-1, jstar[..., None], float("-inf"))
    gap = ks.norm(dim=-1) - proj.amax(-1)   # +inf when Lk == 1
    gap = torch.where(torch.isinf(gap), ks.norm(dim=-1), gap)
    c = PEAK_GAP * 1.001 / (SCALE * gap)
    kind = torch.where(((kind == 1) | (kind == 2)) & (c > 64 * math.sqrt(HD)), torch.zeros_like(kind), kind)
    qn = torch.where(((kind == 1) | (kind == 2))[..., None], c[..., None] * us, q)
    # huge-logit
    s = SCALE * torch.einsum("bqhd,bkhd->bqhk", q, k)
    qn = torch.where((kind == 3)[..., None], q * (HUGE_SPAN / s.abs().amax(-1))[..., None], qn)
    # rising, uniform
    qn = torch.where((kind == 4)[..., None], (RISE_SPAN / (4.0 * SCALE)) * u.view(1, 1, heads, HD), qn)
    qn = torch.where((kind == 5)[..., None], torch.zeros_like(qn), qn)
    C = heads * HD
    return qn.reshape(B, Lq, C).to(dtype), k.reshape(B, Lk, C).to(dtype), v.reshape(B, Lk, C).to(dtype), kind


MASK_KINDS = ("random", "none_allowed", "one_allowed", "leading_masked", "alternating", "all_allowed")


def make_mask(B, Lq, Lk, seed, LkP=None, pad=1):
    """(uint8 mask [B, Lq, LkP] with 1 = key not allowed, int32 allowed-key counts [B, Lq]); LkP defaults to round4(Lk), bytes Lk..LkP hold `pad`.
    Row r (flattened over the batch) has kind r % 6; the one-allowed rows cycle the allowed key through 0, Lk-1 and both sides of the 64 / 128 / 256
    boundaries, the leading-masked rows the number of masked leading keys through 64, 128, 256, 512 and Lk-1 (then 30% of the rest masked)."""
    LkP = (Lk + 3) // 4 * 4 if LkP is None else LkP
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand((B * Lq, Lk), generator=g) < 0.5).to(torch.uint8)
    one = [j for j in (0, Lk - 1, 63, 64, 127, 128, 255, 256) if j < Lk]
    lead = [n for n in (64, 128, 256, 512, Lk - 1) if 0 < n < Lk] or [0]
    keys = torch.arange(Lk)
    for r in range(B * Lq):
        t, n = r % 6, r // 6
        if t == 1:
            m[r] = 1
        elif t == 2:
            m[r] = 1
            m[r, one[n % len(one)]] = 0
        elif t == 3:
            m[r] = (torch.rand(Lk, generator=g) < 0.3).to(torch.uint8)
            m[r, :lead[n % len(lead)]] = 1
        elif t == 4:
            m[r] = ((keys + n) % 2).to(torch.uint8)
        elif t == 5:
            m[r] = 0
    mask = torch.full((B * Lq, LkP), pad, dtype=torch.uint8)
    mask[:, :Lk] = m
    allowed = (m == 0).sum(-1).to(torch.int32)
    return mask.view(B, Lq, LkP), allowed.view(B, Lq)


# ---- the fp64 reference itself (no GPU) -----------------------------------------------------------------------------------------------------------------------
def test_attention_reference_self_check():
    B, Lq, Lk, heads = 2, 97, 300, 2
    q, k, v, kind = make_qkv(B, Lq, Lk, heads, 1)
    ref = RefBackend()
    # the generator: every kind of row, with the properties the file states
    assert set(kind.unique().tolist()) == set(range(len(KINDS)))
    P = probs64(q, k, heads, SCALE)
    s = SCALE * _split_heads(q, heads) @ _split_heads(k, heads).transpose(-1, -2)
    kt = kind.transpose(1, 2)
    top2 = s.topk(2, -1).values
    peaked = (kt == 1) | (kt == 2)
    assert bool((top2[..., 0] - top2[..., 1])[peaked].min() >= 30)
    arg = s.argmax(-1)
    assert bool((arg[kt == 1] < 64).all() and (arg[kt == 2] >= (Lk - 1) // 64 * 64).all())
    huge = s[kt == 3]
    assert bool((huge.abs().amax(-1) - HUGE_SPAN).abs().max() < 1e-3) and bool((huge.amin(-1) < -HUGE_SPAN / 4).all())
    assert float(((huge - huge.amax(-1, keepdim=True)) < -87.3).to(F64).mean()) > 0.2   # exp underflows past the fp32 normal range
    rising = s[kt == 4]
    assert bool((rising[..., 1:] > rising[..., :-1]).all())
    assert bool((P[kt == 5] == 1.0 / Lk).all())
    # fp32 computations of the same graph stay inside the forward and gradient bounds (RefBackend: torch in fp32)
    want, bound = out_bound(q, k, v, heads, SCALE, kind)
    out32 = torch.empty_like(q)
    ref.attention(q, k, v, out32, heads, SCALE)
    assert_within(out32, want, bound, "RefBackend.attention vs fp64")
    dout = torch.randn(q.shape, generator=torch.Generator().manual_seed(2))
    o64 = attn64(q, k, v, heads, SCALE)
    grads, gb = grad_bounds(q, k, v, o64.float(), dout, heads, SCALE, kind)
    g32 = [torch.empty_like(t) for t in (q, k, v)]
    ref.attention_bwd(q, k, v, o64.float(), dout, heads, SCALE, *g32)
    for got, w, b, name in zip(g32, grads, gb, ("dq", "dk", "dv")):
        assert_within(got, w, b, f"RefBackend.attention_bwd {name} vs fp64")
    # the written-out backward equals fp64 autograd of the forward
    leaves = [t.to(F64).requires_grad_(True) for t in (q, k, v)]
    auto = torch.autograd.grad(attn64(*leaves, heads, SCALE), leaves, dout.to(F64))
    for a, b, name in zip(auto, grads, ("dq", "dk", "dv")):
        assert_within(b, a, 1e-12 * float(a.abs().max()), f"attn_bwd64 {name} vs fp64 autograd")
    # masked: against RefBackend.attention_masked and F.scaled_dot_product_attention in float64 with a boolean mask (True = takes part)
    mask, allowed = make_mask(B, Lq, Lk, 3, LkP=Lk + 8, pad=0)
    assert bool((allowed[mask[:, :, :Lk].all(-1).bool()] == 0).all())
    want, bound = out_bound(q, k, v, heads, SCALE, kind, mask)
    ref.attention_masked(q, k, v, mask, allowed, out32, heads, SCALE)
    assert_within(out32, want, bound, "RefBackend.attention_masked vs fp64")
    keep = (mask[:, :, :Lk] == 0) | (allowed == 0)[..., None]
    sdpa = F.scaled_dot_product_attention(*(_split_heads(t, heads) for t in (q, k, v)), attn_mask=keep[:, None], scale=SCALE)
    assert_within(_merge_heads(sdpa), want, 1e-12 * float(want.abs().max()), "F.scaled_dot_product_attention vs fp64")
    # a row with no allowed key attends everywhere, one with a single allowed key returns that key's value
    none = allowed == 0
    assert bool(none.any()) and torch.equal(want[none], attn64(q, k, v, heads, SCALE)[none])
    r1 = (allowed == 1).nonzero()
    b_, r = (int(x) for x in r1[0])
    j = int((mask[b_, r, :Lk] == 0).nonzero()[0])
    assert torch.equal(want[b_, r], v[b_, j].to(F64))
    # the mask generator reaches every kind of row, and every one-allowed position
    for n, j in enumerate((0, Lk - 1, 63, 64, 127, 128, 255, 256)):
        r = 2 + 6 * n
        assert int(allowed.view(-1)[r]) == 1 and int(mask.view(-1, Lk + 8)[r, j]) == 0


# ---- GPU helpers ---------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def be():
    """the CUDA backend (never the CPU reference backend some host-graph tests install)"""
    b = ops._be()
    assert isinstance(b, ops.CudaBackend)
    return b


def _view(t, width, at, fill=NAN):
    """t as the column slice [at, at + C) of a wider buffer whose other columns hold `fill`"""
    buf = torch.full((*t.shape[:-1], width), fill, dtype=t.dtype, device=t.device)
    buf[..., at:at + t.shape[-1]] = t
    return buf[..., at:at + t.shape[-1]]


# how each dispatch path is reached: (dtype, layout of q / k / v)
PATHS = {
    "f32": (torch.float32, None),
    "f16_tc": (torch.float16, None),
    "f16_simt_pitch": (torch.float16, "pitch"),   # rows C + 4 halves apart (260 at 8 heads): not a multiple of 8
    "f16_simt_off8": (torch.float16, "off8"),     # rows start 8 bytes past a 16-byte boundary
    "split_f32": (torch.float32, None),
    "split_pair": (torch.float32, None),
}


def _layout(t, how):
    C = t.shape[-1]
    if how == "pitch":
        return _view(t, C + 4, 0)
    if how == "off8":
        return _view(t, C + 8, 4)
    return t.contiguous()


def run_attention(be, path, q, k, v, heads, scale=SCALE):
    """fb200_attention / fb200_attention_split on the path's layout; returns the output as float64 ([hi | lo] pairs: hi + lo, after checking that
    lo is the fp16 remainder of hi)"""
    how = PATHS[path][1]
    qd, kd, vd = (_layout(t.to(DEV), how) for t in (q, k, v))
    if path == "split_pair":
        out = ops.Pair(torch.full((*q.shape[:-1], 2 * q.shape[-1]), NAN, dtype=torch.float16, device=DEV))
        be.attention(qd, kd, vd, out, heads, scale, True)
        hi, lo = out.hi.to(F64), out.lo.to(F64)
        assert bool((lo.abs() <= 2.0 ** -11 * hi.abs() + 2.0 ** -25).all()), "lo is not the fp16 remainder of hi"
        return hi + lo
    out = torch.full(q.shape, NAN, dtype=q.dtype, device=DEV)
    be.attention(qd, kd, vd, out, heads, scale, path.startswith("split"))
    return out.to(F64)


def run_masked(be, path, q, k, v, mask, allowed, heads, scale=SCALE):
    """fb200_attention_masked / fb200_attention_masked_split; the split paths take K / V as fp32 tensors or as the [hi | lo] pairs of their values"""
    how = PATHS[path][1]
    qd, kd, vd = (_layout(t.to(DEV), how) for t in (q, k, v))
    md, ad = mask.to(DEV), allowed.to(DEV)
    out = torch.full(q.shape, NAN, dtype=q.dtype, device=DEV)
    if path == "split_pair":
        be.attention_masked_split(qd, ops.Pair(ops.split_pair(kd)), ops.Pair(ops.split_pair(vd)), md, ad, out, heads, scale)
    elif path == "split_f32":
        be.attention_masked_split(qd, kd, vd, md, ad, out, heads, scale)
    else:
        be.attention_masked(qd, kd, vd, md, ad, out, heads, scale)
    return out.to(F64)


def attention_kernels(prof):
    """names of the attention kernels a torch.profiler session recorded, in launch order"""
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "attention" in e.name]
    return [e.name for e in sorted(ev, key=lambda e: e.time_range.start)]


# shapes: (B, Lq, Lk, heads)
SHIPPED = {
    "detr_aifi_400": (2, 400, 400, 8), "detr_decoder_self_300": (2, 300, 300, 8),
    "mf_encoder_400": (1, 400, 400, 8), "mf_encoder_625": (1, 625, 625, 8), "mf_encoder_768": (1, 768, 768, 8), "mf_encoder_1024": (1, 1024, 1024, 8),
    "mf_decoder_self_100": (2, 100, 100, 8),
}
LQS = (1, 15, 16, 17, 63, 64, 65, 191, 192, 193)              # 16-row warp tile, 64-query CTA, 192-query split block
LKS = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257)        # 64-key MMA block, 128 / 256-key stream chunks
# every Lq twice and every Lk at least once, mostly Lq != Lk in both directions; heads 1 and 8, B 1..4
TAILS = [(1 + i % 4, lq, LKS[(i * 3 + j * 5) % len(LKS)], 8 if (i + j) % 2 else 1) for i, lq in enumerate(LQS) for j in range(2)]
MASKED_SHIPPED = {   # Lq = 100 queries of the masked decoders against the keys of one feature level
    "mf_640_l0": (2, 100, 400, 8), "mf_640_l1": (2, 100, 1600, 8), "mf_640_l2": (1, 100, 6400, 8),
    "mf_1024_l0": (2, 100, 1024, 8), "mf_1024_l1": (1, 100, 4096, 8), "mf_1024_l2": (1, 100, 16384, 8),
    "bisenetformer_1024x512_l0": (2, 100, 512, 8), "bisenetformer_1024x512_l1": (1, 100, 2048, 8),
}


def _check_forward(be, path, B, Lq, Lk, heads, seed):
    dtype = PATHS[path][0]
    q, k, v, kind = make_qkv(B, Lq, Lk, heads, seed, dtype)
    want, bound = out_bound(q.to(DEV), k.to(DEV), v.to(DEV), heads, SCALE, kind.to(DEV), f16=dtype == torch.float16)
    assert_within(run_attention(be, path, q, k, v, heads), want, bound, f"{path} B={B} Lq={Lq} Lk={Lk} heads={heads}")


# ---- forward -----------------------------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("path", list(PATHS))
def test_attention_forward_shipped_shapes(be, path):
    for n, (name, (B, Lq, Lk, heads)) in enumerate(SHIPPED.items()):
        if path == "split_pair" and Lk > 640:
            continue   # pair rows stop at the resident kernel (test_attention_ceilings)
        _check_forward(be, path, B, Lq, Lk, heads, 100 + n)


@gpu
@pytest.mark.parametrize("path", list(PATHS))
def test_attention_forward_tails(be, path):
    for n, (B, Lq, Lk, heads) in enumerate(TAILS):
        _check_forward(be, path, B, Lq, Lk, heads, 200 + n)
        _check_forward(be, path, B, Lk, Lq, heads, 300 + n)   # the other direction


MASKED_PATHS = ("f32", "f16_tc", "f16_simt_pitch", "split_f32", "split_pair")


def _check_masked(be, path, B, Lq, Lk, heads, seed, LkP=None, pad=1):
    dtype = PATHS[path][0]
    q, k, v, kind = make_qkv(B, Lq, Lk, heads, seed, dtype)
    mask, allowed = make_mask(B, Lq, Lk, seed + 1, LkP, pad)
    want, bound = out_bound(q.to(DEV), k.to(DEV), v.to(DEV), heads, SCALE, kind.to(DEV), mask.to(DEV), f16=dtype == torch.float16)
    got = run_masked(be, path, q, k, v, mask, allowed, heads)
    assert_within(got, want, bound, f"masked {path} B={B} Lq={Lq} Lk={Lk} LkP={mask.shape[2]} pad={pad} heads={heads}")


@gpu
@pytest.mark.parametrize("path", MASKED_PATHS)
def test_attention_masked_shipped_shapes(be, path):
    for n, (B, Lq, Lk, heads) in enumerate(MASKED_SHIPPED.values()):
        _check_masked(be, path, B, Lq, Lk, heads, 400 + 2 * n)


@gpu
@pytest.mark.parametrize("path", MASKED_PATHS)
def test_attention_masked_tails_and_zero_padding(be, path):
    """the tail shapes in both directions; every other case with a mask row pitch 8 bytes past round4(Lk) whose padding bytes are 0 (not keys:
    the kernels must bound keys by Lk, not by the mask)"""
    for n, (B, Lq, Lk, heads) in enumerate(TAILS):
        for m, (lq, lk) in enumerate(((Lq, Lk), (Lk, Lq))):
            zero_pad = (n + m) % 2 == 0
            LkP = (lk + 3) // 4 * 4 + 8 if zero_pad else None
            _check_masked(be, path, B, lq, lk, heads, 500 + 4 * n + 2 * m, LkP, 0 if zero_pad else 1)


# ---- backward ----------------------------------------------------------------------------------------------------------------------------------------------------------
def _check_grads(dq, dk, dv, q, k, v, o, dout, heads, kind, what):
    grads, bounds = grad_bounds(q, k, v, o, dout, heads, SCALE, kind)
    for got, w, b, name in zip((dq, dk, dv), grads, bounds, ("dq", "dk", "dv")):
        assert_within(got, w, b, f"{what}: {name}")


@gpu
@pytest.mark.parametrize("split", [False, True], ids=["fp32", "split"])
@pytest.mark.parametrize("L", [300, 400])
def test_attention_fn_training_shapes(be, L, split):
    """AttentionFn as the fine-tune step runs it (B = 4; split in the fp32_tc and amp precisions): forward and fp64-autograd gradients"""
    B, heads = 4, 8
    q, k, v, kind = (t.to(DEV) for t in make_qkv(B, L, L, heads, 600 + L + split))
    dout = torch.randn(q.shape, generator=torch.Generator().manual_seed(L), dtype=torch.float32).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    y = A.AttentionFn.apply(*leaves, heads, SCALE, split)
    y.backward(dout)
    want, bound = out_bound(q, k, v, heads, SCALE, kind)
    assert_within(y, want, bound, f"AttentionFn L={L} split={split}: out")
    _check_grads(*(t.grad for t in leaves), q, k, v, y.detach(), dout, heads, kind, f"AttentionFn L={L} split={split}")


@gpu
def test_attention_bwd_tails(be):
    """fb200_attention_bwd at the tail shapes in both directions, heads 1 and 8"""
    for n, (B, Lq, Lk, heads) in enumerate(TAILS):
        for lq, lk in ((Lq, Lk), (Lk, Lq)):
            q, k, v, kind = (t.to(DEV) for t in make_qkv(B, lq, lk, heads, 700 + n))
            dout = torch.randn(q.shape, generator=torch.Generator().manual_seed(n), dtype=torch.float32).to(DEV)
            o = attn64(q, k, v, heads, SCALE).float()
            g = [torch.full_like(t, NAN) for t in (q, k, v)]
            be.attention_bwd(q, k, v, o, dout, heads, SCALE, *g)
            _check_grads(*g, q, k, v, o, dout, heads, kind, f"attention_bwd B={B} Lq={lq} Lk={lk} heads={heads}")


# ---- ABI ----------------------------------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("path", ["f32", "f16_tc", "split_f32", "split_pair", "masked_f16_tc", "masked_split_f32"])
def test_attention_abi_slices_sentinels_determinism_batch_invariance(be, path):
    """q and k as the two column halves of the fused qk projection and v as a slice of a wider buffer (every other column NaN); the output a slice
    of a buffer whose other columns hold a sentinel; two calls give the same bits, and image b gives the same bits alone and in a batch of 4"""
    B, L, heads = 4, 300, 8
    C = heads * HD
    masked = path.startswith("masked")
    dtype = torch.float16 if "f16" in path else torch.float32
    q, k, v, kind = (t.to(DEV) for t in make_qkv(B, L, L, heads, 800, dtype))
    qk = torch.full((B, L, 2 * C + 16), NAN, dtype=dtype, device=DEV)
    qk[..., :C], qk[..., C:2 * C] = q, k
    qs, ks, vs = qk[..., :C], qk[..., C:2 * C], _view(v, C + 64, 32)
    mask, allowed = (t.to(DEV) for t in make_mask(B, L, L, 801))
    pair = path == "split_pair"
    width = 2 * C + 48 if pair else C + 48

    def call(b0, b1):
        buf = torch.full((b1 - b0, L, width), 7.0, dtype=torch.float16 if pair else dtype, device=DEV)
        if pair:
            out = ops.Pair(buf[..., 16:16 + 2 * C])
            be.attention(qs[b0:b1], ks[b0:b1], vs[b0:b1], out, heads, SCALE, True)
        elif masked:
            out = buf[..., 16:16 + C]
            if path == "masked_split_f32":
                be.attention_masked_split(qs[b0:b1], ks[b0:b1], vs[b0:b1], mask[b0:b1], allowed[b0:b1], out, heads, SCALE)
            else:
                be.attention_masked(qs[b0:b1], ks[b0:b1], vs[b0:b1], mask[b0:b1], allowed[b0:b1], out, heads, SCALE)
        else:
            be.attention(qs[b0:b1], ks[b0:b1], vs[b0:b1], buf[..., 16:16 + C], heads, SCALE, path == "split_f32")
        torch.cuda.synchronize()
        return buf

    first, second = call(0, B), call(0, B)
    assert torch.equal(first, second), f"{path}: two calls differ"
    assert bool((first[..., :16] == 7).all() and (first[..., width - 32:] == 7).all()), f"{path}: columns outside the output slice were written"
    got = (first[..., 16:16 + C].to(F64) + first[..., 16 + C:16 + 2 * C].to(F64)) if pair else first[..., 16:16 + C].to(F64)
    want, bound = out_bound(q, k, v, heads, SCALE, kind, mask if masked else None, f16=dtype == torch.float16)
    assert_within(got, want, bound, f"{path} on slices")
    for b in (0, 3):
        assert torch.equal(call(b, b + 1)[0], first[b]), f"{path}: image {b} differs between a batch of 1 and a batch of 4"


@gpu
def test_attention_bwd_abi_slices_sentinels_determinism_batch_invariance(be):
    """fb200_attention_bwd through the backend: q, k from the fused qk projection, v, o and dout as slices of NaN-padded buffers, dq / dk / dv as
    slices of buffers whose other columns keep a sentinel; bitwise identical across calls and between a batch of 1 and a batch of 4"""
    B, L, heads = 4, 300, 8
    C = heads * HD
    q, k, v, kind = (t.to(DEV) for t in make_qkv(B, L, L, heads, 900))
    dout = torch.randn(q.shape, generator=torch.Generator().manual_seed(901)).to(DEV)
    o = attn64(q, k, v, heads, SCALE).float()
    qk = torch.full((B, L, 2 * C + 16), NAN, device=DEV)
    qk[..., :C], qk[..., C:2 * C] = q, k
    ins = (qk[..., :C], qk[..., C:2 * C], _view(v, C + 64, 32), _view(o, C + 8, 4), _view(dout, C + 40, 8))

    def call(b0, b1):
        bufs = [torch.full((b1 - b0, L, C + 48), 7.0, device=DEV) for _ in range(3)]
        be.attention_bwd(*(t[b0:b1] for t in ins), heads, SCALE, *(bf[..., 16:16 + C] for bf in bufs))
        torch.cuda.synchronize()
        return bufs

    first, second = call(0, B), call(0, B)
    for a, b, name in zip(first, second, ("dq", "dk", "dv")):
        assert torch.equal(a, b), f"{name}: two calls differ"
        assert bool((a[..., :16] == 7).all() and (a[..., 16 + C:] == 7).all()), f"{name}: columns outside the slice were written"
    _check_grads(*(bf[..., 16:16 + C] for bf in first), q, k, v, o, dout, heads, kind, "attention_bwd on slices")
    for b in (1, 2):
        for a, full, name in zip(call(b, b + 1), first, ("dq", "dk", "dv")):
            assert torch.equal(a[0], full[b]), f"{name}: image {b} differs between a batch of 1 and a batch of 4"


# ---- shared-memory ceilings ----------------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_attention_ceilings(be):
    """Each resident kernel at the largest key count whose K and V fit 227 KiB of shared memory, and one key past it, where the entry point takes
    the streaming kernel (or, for pair output and the backward, refuses without a launch)"""
    cases = [   # (path, Lq, Lk, kernel expected)
        ("f32", 792, 792, r"\battention_kernel<float>"), ("f32", 793, 793, r"\battention_masked_kernel<float>"),
        ("f16_simt_pitch", 792, 792, r"\battention_kernel<__half>"), ("f16_simt_off8", 793, 793, r"\battention_masked_kernel<__half>"),
        ("f16_tc", 1408, 1408, r"\battention_mma_kernel\b"), ("f16_tc", 1409, 1409, r"\battention_mma_stream_kernel\b"),
        ("split_f32", 640, 640, r"\battention_mma_split_kernel\b"), ("split_f32", 641, 641, r"\battention_mma_split_stream_kernel<false>"),
        ("split_f32", 32, 704, r"\battention_mma_split_kernel\b"), ("split_f32", 32, 705, r"\battention_mma_split_stream_kernel<false>"),
        ("split_pair", 640, 640, r"\battention_mma_split_kernel\b"), ("split_pair", 32, 704, r"\battention_mma_split_kernel\b"),
    ]
    bwd_cases = ((398, r"attention_bwd_kernel<36>"), (399, r"attention_bwd_kernel<33>"), (433, r"attention_bwd_kernel<33>"))
    from torch.profiler import ProfilerActivity, profile

    results = []
    # kernels launched right as a session starts have been seen missing from its trace, after a long run of other GPU tests in the same process: every
    # path runs once before the session (its kernel loaded), and the session opens with a kernel of no interest that has finished before the work starts
    for n, (path, Lq, Lk, kernel) in enumerate(cases):
        run_attention(be, path, *make_qkv(1, Lq, Lk, 4, 1000 + n, PATHS[path][0])[:3], 4)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:   # one session; each call launches one attention kernel
        torch.ones(1, device=DEV).add_(1)
        torch.cuda.synchronize()
        time.sleep(0.2)
        for n, (path, Lq, Lk, kernel) in enumerate(cases):
            q, k, v, kind = make_qkv(1, Lq, Lk, 4, 1000 + n, PATHS[path][0])
            results.append((run_attention(be, path, q, k, v, 4), q, k, v, kind))
        for L, kernel in bwd_cases:
            q, k, v, kind = (t.to(DEV) for t in make_qkv(1, L, L, 4, 1100 + L))
            dout = torch.randn(q.shape, generator=torch.Generator().manual_seed(L)).to(DEV)
            o = attn64(q, k, v, 4, SCALE).float()
            g = [torch.full_like(t, NAN) for t in (q, k, v)]
            be.attention_bwd(q, k, v, o, dout, 4, SCALE, *g)
            results.append((g, q, k, v, kind, o, dout))
        torch.cuda.synchronize()
    names = attention_kernels(prof)
    expected = [(c[3], f"{c[0]} Lq={c[1]} Lk={c[2]}") for c in cases] + [(kernel, f"attention_bwd L={L}") for L, kernel in bwd_cases]
    assert len(names) == len(expected), f"{len(names)} attention kernels launched for {len(expected)} calls: {names}"
    for name, (pattern, what) in zip(names, expected):
        assert re.search(pattern, name), f"{what}: expected {pattern}, launched {name}"
    for (path, Lq, Lk, _), (got, q, k, v, kind) in zip(cases, results):
        want, bound = out_bound(q.to(DEV), k.to(DEV), v.to(DEV), 4, SCALE, kind.to(DEV), f16=PATHS[path][0] == torch.float16)
        assert_within(got, want, bound, f"ceiling {path} Lq={Lq} Lk={Lk}")
    for (L, _), (g, q, k, v, kind, o, dout) in zip(bwd_cases, results[len(cases):]):
        _check_grads(*g, q, k, v, o, dout, 4, kind, f"attention_bwd ceiling L={L}")
    # pair rows one key past the resident kernel: refused, nothing written
    for Lq, Lk in ((641, 641), (32, 705)):
        q, k, v = (torch.randn((1, L, 128), device=DEV) for L in (Lq, Lk, Lk))
        out = ops.Pair(torch.full((1, Lq, 256), 7.0, dtype=torch.float16, device=DEV))
        with pytest.raises(RuntimeError, match=r"\(-2\).*does not fit shared memory"):
            be.attention(q, k, v, out, 4, SCALE, True)
        torch.cuda.synchronize()
        assert bool((out.buf == 7).all())
    # backward: the float4 layout up to L = 398, the 33-float layout up to 433 (checked above), refused at 434
    t = torch.randn((1, 434, 128), device=DEV)
    g = [torch.full_like(t, 7.0) for _ in range(3)]
    with pytest.raises(RuntimeError, match=r"\(-1\).*shared-memory-resident"):
        be.attention_bwd(t, t, t, t, t, 4, SCALE, *g)
    torch.cuda.synchronize()
    assert all(bool((x == 7).all()) for x in g)


# ---- argument checks ---------------------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_attention_argument_checks(be):
    """non-positive sizes, pitches below heads*32 and a mask row shorter than Lk are refused on the host, naming the argument, before any launch
    (every buffer is large enough for the launch the bad arguments would describe, and the outputs keep their sentinel)"""
    heads, L = 2, 16
    C = heads * HD
    x = torch.randn((4, L, 2 * C), device=DEV)
    p = x.data_ptr()
    out = torch.full((4, L, 2 * C), 7.0, device=DEV)
    o = out.data_ptr()
    mask = torch.zeros((4, L, 2 * L), dtype=torch.uint8, device=DEV)
    allowed = torch.full((4, L), L, dtype=torch.int32, device=DEV)
    st = ops._stream()
    f32 = ops.F32

    def fwd(B=4, Lq=L, Lk=L, h=heads, qp=C, kp=C, vp=C, op=C):
        be._call("fb200_attention", p, qp, p, kp, p, vp, o, op, f32, B, Lq, Lk, h, HD, SCALE, st)

    def split(B=4, Lq=L, Lk=L, h=heads, qp=C, kp=C, vp=C, op=C):
        be._call("fb200_attention_split", p, qp, p, kp, p, vp, o, f32, op, B, Lq, Lk, h, HD, SCALE, st)

    def masked(B=4, Lq=L, Lk=L, h=heads, qp=C, kp=C, vp=C, op=C, LkP=L):
        be._call("fb200_attention_masked", p, qp, p, kp, p, vp, mask.data_ptr(), LkP, allowed.data_ptr(), o, op, f32, B, Lq, Lk, h, HD, SCALE, st)

    def bwd(B=4, Lq=L, Lk=L, h=heads, qp=C, kp=C, vp=C, op=C, dop=C, dqp=C, dkp=C, dvp=C):
        be._call("fb200_attention_bwd", p, qp, p, kp, p, vp, p, op, p, dop, B, Lq, Lk, h, HD, SCALE, o, dqp, o, dkp, o, dvp, st)

    entries = {"attention": (fwd, ("q_pitch", "k_pitch", "v_pitch", "out_pitch")), "attention_split": (split, ("q_pitch", "k_pitch", "v_pitch", "out_pitch")),
               "attention_masked": (masked, ("q_pitch", "k_pitch", "v_pitch", "out_pitch")),
               "attention_bwd": (bwd, ("q_pitch", "k_pitch", "v_pitch", "o_pitch", "do_pitch", "dq_pitch", "dk_pitch", "dv_pitch"))}
    kw = {"q_pitch": "qp", "k_pitch": "kp", "v_pitch": "vp", "out_pitch": "op", "o_pitch": "op", "do_pitch": "dop", "dq_pitch": "dqp", "dk_pitch": "dkp", "dv_pitch": "dvp"}
    for name, (fn, pitches) in entries.items():
        for arg in ("B", "Lq", "Lk", "h"):
            for bad in (0, -1):
                with pytest.raises(RuntimeError, match=rf"\(-1\).*{name}: B, Lq, Lk and heads must be positive"):
                    fn(**{arg: bad})
        for pitch in pitches:
            with pytest.raises(RuntimeError, match=rf"\(-1\).*{name}: {pitch} \({C - 4}\) < heads\*32 \({C}\)"):
                fn(**{kw[pitch]: C - 4})
    with pytest.raises(RuntimeError, match=r"\(-1\).*attention_masked: LkP \(12\) < Lk \(16\)"):
        masked(LkP=12)
    torch.cuda.synchronize()
    assert bool((out == 7).all())
