"""Multi-scale deformable attention, forward (`fb200_msda`, csrc/msda.cu) and backward (`fb200_msda_bwd`, csrc/bwd_attn.cu), against a float64
reference built on F.grid_sample.

The sampling points are placed on purpose: inside the maps, straddling each of the four borders (ix, iy in (-1, 0) and (W-1, W)), fully outside,
a few map widths outside, and in the whole-pixel case exactly on pixel centres.  The logit rows mix random, large (+-50), all-equal and one-dominant
rows.  Forward: every dtype path `fb200_msda` dispatches to, the vector kernel on a column slice of the fused value projection and the scalar kernel
on rows that are not 8/16-byte aligned.  Backward: `dvalue` and `doa` against fp64 autograd, and the ABI contract of the backward entry point.

Tolerances are relative to the scale (max |.|) of the fp64 result: FWD_TOL for fp32 outputs, one fp16 rounding more for fp16 outputs, 5e-5 for
each gradient.  Where the fp64 result is exactly zero (no in-map corner), the kernels must give exactly zero.

`test_fp64_reference_self_check` needs no GPU: it checks the fp64 reference before any GPU test relies on it."""
import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import autograd_ops as A
from focoos_b200 import ops
from oracle.ops_ref import RefBackend

pytestmark = pytest.mark.timeout(600)
gpu = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
# the fp32 rounding of a sampling position alone (ulp of loc ~ 1, times W = 80 pixels, times the value step between two pixels) reaches 1e-5 of
# the output scale at the 80x80 level
FWD_TOL = 2e-5

SHIPPED = [(20, 20), (40, 40), (80, 80)]   # the decoder's levels at 640x640, in the model's order
CASES = {  # name: (B, Q, heads, P, level shapes, seed)
    "shipped_640": (2, 300, 8, 4, SHIPPED, 1),
    "non_square": (2, 120, 8, 4, [(48, 80), (24, 40), (12, 20)], 2),
    "odd": (3, 77, 8, 4, [(25, 38), (13, 19), (7, 10)], 3),
    "one_level_one_point": (2, 64, 8, 1, [(33, 47)], 4),
    "four_levels_8_points": (2, 64, 4, 8, [(32, 48), (16, 24), (8, 12), (4, 6)], 5),   # L*P = 32: the whole warp, the largest accepted
}
BWD_CASES = dict(CASES, finetune_b4=(4, 300, 8, 4, SHIPPED, 6))
DYADIC_SHAPES = [(16, 16), (32, 32), (8, 8)]


# ---- float64 reference ---------------------------------------------------------------------------------------------------------------------------------
def _weights_and_locations(oa, ref, L, P, heads):
    """softmax weights [B,Q,heads,L,P] over the L*P logits of a head and sampling locations [B,Q,heads,L,P,2] (x, y in [0, 1] map units)"""
    B, Q = oa.shape[:2]
    off = oa[..., :heads * L * P * 2].reshape(B, Q, heads, L, P, 2)
    w = torch.softmax(oa[..., heads * L * P * 2:heads * L * P * 3].reshape(B, Q, heads, L * P), -1).reshape(B, Q, heads, L, P)
    r = ref.reshape(B, Q, 1, 1, 1, 4)
    return w, r[..., :2] + off / P * r[..., 2:] * 0.5   # the kernels' association order


def msda64(value, oa, ref, shapes, P, heads):
    """value [B,S,heads*32], oa [B,Q,heads*L*P*3] (offsets, then logits), ref [B,Q,4] -> [B,Q,heads*32], all in float64;
    bilinear zero-padded sampling by F.grid_sample(align_corners=False) per level"""
    value, oa, ref = value.to(F64), oa.to(F64), ref.to(F64)
    B, S, C = value.shape
    Q, L, hd = oa.shape[1], len(shapes), C // heads
    w, loc = _weights_and_locations(oa, ref, L, P, heads)
    out, start = 0, 0
    for l, (H, W) in enumerate(shapes):
        v = value[:, start:start + H * W].reshape(B, H, W, heads, hd).permute(0, 3, 4, 1, 2).reshape(B * heads, hd, H, W)
        g = (2 * loc[:, :, :, l] - 1).transpose(1, 2).reshape(B * heads, Q, P, 2)
        s = F.grid_sample(v, g, mode="bilinear", padding_mode="zeros", align_corners=False).reshape(B, heads, hd, Q, P)
        out = out + torch.einsum("bhdqp,bqhp->bqhd", s, w[:, :, :, l])
        start += H * W
    return out.reshape(B, Q, C)


def msda64_gather(value, oa, ref, shapes, P, heads, cell=torch.floor):
    """the same operator with the bilinear sampling written out as four zero-padded corner gathers (float64, no grid_sample).  `cell` picks the
    top-left corner from the pixel coordinate: floor (the cell to the right and below at a whole pixel) or another convention to compare with."""
    value, oa, ref = value.to(F64), oa.to(F64), ref.to(F64)
    B, S, C = value.shape
    Q, L, hd = oa.shape[1], len(shapes), C // heads
    w, loc = _weights_and_locations(oa, ref, L, P, heads)
    vals = value.reshape(B, S, heads, hd)
    bi, hi = torch.arange(B).view(B, 1, 1, 1), torch.arange(heads).view(1, 1, heads, 1)
    out, start = 0, 0
    for l, (H, W) in enumerate(shapes):
        ix, iy = loc[:, :, :, l, :, 0] * W - 0.5, loc[:, :, :, l, :, 1] * H - 0.5
        x0, y0 = cell(ix), cell(iy)
        tx, ty = ix - x0, iy - y0
        s = 0
        for dx, dy, cw in ((0, 0, (1 - tx) * (1 - ty)), (1, 0, tx * (1 - ty)), (0, 1, (1 - tx) * ty), (1, 1, tx * ty)):
            x, y = x0 + dx, y0 + dy
            inside = (x >= 0) & (x < W) & (y >= 0) & (y < H)
            idx = start + (y.clamp(0, H - 1) * W + x.clamp(0, W - 1)).long()
            s = s + vals[bi, idx, hi] * (cw * inside)[..., None]
        out = out + (s * w[:, :, :, l, :, None]).sum(3)
        start += H * W
    return out.reshape(B, Q, C)


def fwd_bwd64(value, oa, ref, dout, shapes, P, heads, fn=msda64):
    """fp64 output and the autograd gradients w.r.t. value and oa"""
    v, o = value.to(F64).requires_grad_(True), oa.to(F64).requires_grad_(True)
    out = fn(v, o, ref, shapes, P, heads)
    dv, doa = torch.autograd.grad(out, (v, o), dout.to(F64))
    return out.detach(), dv, doa


def pixel_coords64(oa, ref, shapes, P, heads):
    """the fp64 pixel coordinates ix, iy [B,Q,heads,L,P] that grid_sample and the kernels sample at"""
    L = len(shapes)
    _, loc = _weights_and_locations(oa.to(F64), ref.to(F64), L, P, heads)
    H, W = (torch.tensor([s[i] for s in shapes], dtype=F64).view(1, 1, 1, L, 1) for i in (0, 1))
    g = 2 * loc - 1
    return ((g[..., 0] + 1) * W - 1) * 0.5, ((g[..., 1] + 1) * H - 1) * 0.5


# ---- inputs ----------------------------------------------------------------------------------------------------------------------------------------------
# placement of a point along one axis of n pixels, as a pixel-coordinate range: inside, straddling the low / high border, fully outside low / high,
# and 1-9 map widths outside (|loc| <= 10)
KIND_P = [0.6, 0.1, 0.1, 0.05, 0.05, 0.05, 0.05]


def _axis(kind, n, u):
    z = torch.zeros_like(n)
    lo = torch.stack(torch.broadcast_tensors(z, z - 1, n - 1, z - 3, n, -9 * n - 0.5, 2 * n - 0.5), -1)
    hi = torch.stack(torch.broadcast_tensors(n - 1, z, n, z - 1, n + 2, -n - 0.5, 10 * n - 0.5), -1)
    lo, hi = (t.expand(*kind.shape, 7).gather(-1, kind.unsqueeze(-1)).squeeze(-1) for t in (lo, hi))
    return lo + (hi - lo) * u


def _logit_rows(shape, g):
    """logit rows of four kinds: random, large (+-50), all equal, one dominant"""
    *lead, LP = shape
    z = torch.randn(shape, generator=g, dtype=F64) * 1.5
    big = (torch.rand(shape, generator=g, dtype=F64) * 2 - 1) * 50
    equal = (torch.randn((*lead, 1), generator=g, dtype=F64) * 3).expand(shape)
    dom = z / 1.5 + 25 * F.one_hot(torch.randint(0, LP, lead, generator=g), LP)
    kind = torch.multinomial(torch.tensor([0.55, 0.15, 0.15, 0.15]), z.numel() // LP, replacement=True, generator=g).view(*lead, 1)
    return torch.where(kind == 0, z, torch.where(kind == 1, big, torch.where(kind == 2, equal, dom)))


def make_inputs(B, Q, heads, shapes, P, seed, v_dtype=torch.float32, oa_dtype=torch.float32, boundary_free=False):
    """(value, oa, ref) on the CPU.  Reference boxes anywhere in the image with widths up to the whole image; each point gets an x and a y
    placement kind (KIND_P), and 3% of the head rows have every point outside their map.  boundary_free: no sampling coordinate lies within 1e-3 of
    a whole pixel in fp64, so fp32 and fp64 always pick the same cell (the offset gradient jumps at whole pixels)."""
    g = torch.Generator().manual_seed(seed)
    L, S = len(shapes), sum(h * w for h, w in shapes)
    value = torch.randn((B, S, heads * 32), generator=g).to(v_dtype)
    ref = torch.cat([torch.rand((B, Q, 2), generator=g), 0.05 + 0.95 * torch.rand((B, Q, 2), generator=g)], -1)
    pts = (B, Q, heads, L, P)
    kx, ky = (torch.multinomial(torch.tensor(KIND_P), B * Q * heads * L * P, replacement=True, generator=g).view(pts) for _ in range(2))
    outside_rows = torch.rand((B, Q, heads, 1, 1), generator=g) < 0.03
    kx = torch.where(outside_rows, 3 + torch.randint(0, 4, pts, generator=g), kx)
    ux, uy = torch.rand(pts, generator=g, dtype=F64), torch.rand(pts, generator=g, dtype=F64)
    logits = _logit_rows((B, Q, heads, L * P), g)
    Hs = torch.tensor([h for h, _ in shapes], dtype=F64).view(1, 1, 1, L, 1)
    Ws = torch.tensor([w for _, w in shapes], dtype=F64).view(1, 1, 1, L, 1)
    r = ref.to(F64).view(B, Q, 1, 1, 1, 4)

    def build():
        loc = torch.stack([(_axis(kx, Ws, ux) + 0.5) / Ws, (_axis(ky, Hs, uy) + 0.5) / Hs], -1)
        off = (loc - r[..., :2]) / (r[..., 2:] * 0.5) * P
        return torch.cat([off.reshape(B, Q, -1), logits.reshape(B, Q, -1)], -1).to(oa_dtype)

    oa = build()
    redraws = 0
    while boundary_free:   # redraw the coordinates near a whole pixel (about 0.2% of them per round)
        near_x, near_y = ((t - t.round()).abs() < 1e-3 for t in pixel_coords64(oa, ref, shapes, P, heads))
        if not (near_x.any() or near_y.any()):
            break
        redraws += 1
        assert redraws < 20, "could not draw boundary-free sampling points"
        ux = torch.where(near_x, torch.rand(pts, generator=g, dtype=F64), ux)
        uy = torch.where(near_y, torch.rand(pts, generator=g, dtype=F64), uy)
        oa = build()
    return value, oa, ref


def make_dyadic_inputs(B, Q, heads, shapes, P, seed):
    """(value, oa, ref) whose sampling coordinates are exact in fp32 and fp64: power-of-two levels, ref on a 1/64 grid, widths 1/8, 1/4 or 1/2,
    P = 4, and pixel coordinates k + {0, 1/4, 1/2, 3/4} with k in [-2, W+1].  Most points sit on whole pixels, including -1, 0, W-1 and W."""
    assert P == 4 and all(h & (h - 1) == 0 and w & (w - 1) == 0 and max(h, w) <= 32 for h, w in shapes)
    g = torch.Generator().manual_seed(seed)
    L, S = len(shapes), sum(h * w for h, w in shapes)
    value = torch.randn((B, S, heads * 32), generator=g)
    wh = torch.tensor([0.125, 0.25, 0.5])[torch.randint(0, 3, (B, Q, 2), generator=g)]
    ref = torch.cat([torch.randint(0, 65, (B, Q, 2), generator=g) / 64.0, wh], -1)
    pts = (B, Q, heads, L, P)
    frac = torch.tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.25, 0.5, 0.75], dtype=F64)
    locs = []
    for n_idx in (1, 0):   # x over W, y over H
        n = torch.tensor([s[n_idx] for s in shapes], dtype=F64).view(1, 1, 1, L, 1)
        k = (torch.rand(pts, generator=g, dtype=F64) * (n + 4)).floor() - 2
        locs.append((k + frac[torch.randint(0, 8, pts, generator=g)] + 0.5) / n)
    r = ref.to(F64).view(B, Q, 1, 1, 1, 4)
    off = (torch.stack(locs, -1) - r[..., :2]) / (r[..., 2:] * 0.5) * P
    logits = _logit_rows((B, Q, heads, L * P), g).to(torch.float32).to(F64)
    oa = torch.cat([off.reshape(B, Q, -1), logits.reshape(B, Q, -1)], -1)
    assert torch.equal(oa.to(torch.float32).to(F64), oa), "offsets must be exact in fp32"
    return value, oa.to(torch.float32), ref


# ---- comparisons -----------------------------------------------------------------------------------------------------------------------------------------
def assert_close(got, want, rel, what, f16_out=False):
    """max |got - want| <= rel * max|want| (+ one fp16 rounding of want for fp16 outputs), and exact zeros where want is exactly zero"""
    got, want = got.detach().cpu().to(F64), want.detach().to(F64)
    scale = float(want.abs().max())
    err = (got - want).abs()
    bound = rel * scale + (2.0 ** -11 * want.abs() if f16_out else 0.0)
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, max|d| = {float(err.max()):.3e}, scale {scale:.3e}"
    zero = want == 0
    assert bool((got[zero] == 0).all()), f"{what}: {int((got[zero] != 0).sum())} elements non-zero where the fp64 result is exactly zero"


def check_grads(dvalue, doa, dv64, doa64, heads, L, P, what):
    n_off = heads * L * P * 2
    assert_close(dvalue, dv64, 5e-5, f"{what}: dvalue")
    assert_close(doa[..., :n_off], doa64[..., :n_off], 5e-5, f"{what}: d offsets")
    assert_close(doa[..., n_off:], doa64[..., n_off:], 5e-5, f"{what}: d logits")
    # fully-outside points: no offset gradient, but their logits still take part in the softmax
    out_pts = (doa64[..., :n_off].reshape(*doa64.shape[:2], -1, 2) == 0).all(-1)
    assert bool(out_pts.any()), f"{what}: the case has no fully-outside point"
    if L * P > 1:   # (one point per head: its weight is 1 and its logit gradient 0)
        dlog64 = doa64[..., n_off:].reshape(out_pts.shape)
        assert bool((dlog64[out_pts] != 0).any()) and bool((doa[..., n_off:].cpu().reshape(out_pts.shape)[out_pts] != 0).any())


@pytest.fixture
def be():
    """the CUDA backend (never the CPU reference backend some host-graph tests install)"""
    b = ops._be()
    assert isinstance(b, ops.CudaBackend)
    return b


# ---- the fp64 reference itself (no GPU) --------------------------------------------------------------------------------------------------------------------
def test_fp64_reference_self_check():
    shapes, P, heads = [(25, 38), (13, 19), (7, 10)], 4, 4
    value, oa, ref = make_inputs(2, 40, heads, shapes, P, 11)
    # the generator reaches every placement on each axis of each level: straddling both borders, fully outside, a map width or more outside
    ix, iy = pixel_coords64(oa, ref, shapes, P, heads)
    for l, (H, W) in enumerate(shapes):
        for t, n in ((ix[:, :, :, l], W), (iy[:, :, :, l], H)):
            assert bool(((t > -1) & (t < 0)).any() and ((t > n - 1) & (t < n)).any() and (t < -1).any() and (t > n).any())
            assert bool((t < -n).any() and (t > 2 * n).any())
    # agrees with the fp32 reference backend (RefBackend.msda computes the same graph in fp32)
    out32 = torch.empty((2, 40, heads * 32))
    RefBackend().msda(value, oa, ref, shapes, P, heads, out32)
    want = msda64(value, oa, ref, shapes, P, heads)
    assert_close(out32, want, 1e-5, "RefBackend.msda vs fp64")
    # agrees with the explicit four-gather sampler, output and gradients, at border points and at whole-pixel points
    dy = torch.randn((2, 40, heads * 32), generator=torch.Generator().manual_seed(12))
    dyadic = make_dyadic_inputs(2, 40, heads, DYADIC_SHAPES, 4, 13)
    for (v, o, r), shp, what in (((value, oa, ref), shapes, "border points"), (dyadic, DYADIC_SHAPES, "whole-pixel points")):
        a = fwd_bwd64(v, o, r, dy, shp, 4, heads)
        b = fwd_bwd64(v, o, r, dy, shp, 4, heads, fn=msda64_gather)
        for x, y, name in zip(a, b, ("out", "dvalue", "doa")):
            assert_close(x, y, 1e-12, f"grid_sample vs four gathers at {what}: {name}")
    # at whole pixels grid_sample's offset gradient is the floor one (the cell to the right and below): the cell to the left and above gives the
    # same output but an offset gradient that differs far beyond the GPU tests' tolerance
    v, o, r = dyadic
    a = fwd_bwd64(v, o, r, dy, DYADIC_SHAPES, 4, heads)
    c = fwd_bwd64(v, o, r, dy, DYADIC_SHAPES, 4, heads, fn=lambda *args: msda64_gather(*args, cell=lambda t: torch.ceil(t) - 1))
    assert_close(c[0], a[0], 1e-12, "left-cell convention: out")
    n_off = heads * len(DYADIC_SHAPES) * 4 * 2
    assert float((c[2] - a[2])[..., :n_off].abs().max()) > 100 * 5e-5 * float(a[2][..., :n_off].abs().max())


# ---- forward ---------------------------------------------------------------------------------------------------------------------------------------------
DTYPES = {"f32": (torch.float32, torch.float32), "f16_value_f32_oa": (torch.float16, torch.float32), "f16": (torch.float16, torch.float16)}


@gpu
@pytest.mark.parametrize("dtypes", list(DTYPES))
@pytest.mark.parametrize("case", list(CASES))
def test_msda_forward(be, case, dtypes):
    """every (value, oa, out) combination: the vector kernel on a column slice of the fused six-layer value projection (v_pitch = 6*C, as the
    decoder passes it), the scalar kernel on rows at a pitch of C+2 elements starting one element into the buffer (not 8/16-byte aligned), and for
    fp32 the [hi | lo] fp16 pair output"""
    B, Q, heads, P, shapes, seed = CASES[case]
    v_dt, oa_dt = DTYPES[dtypes]
    f16 = v_dt == torch.float16
    value, oa, ref = make_inputs(B, Q, heads, shapes, P, seed, v_dt, oa_dt)
    want = msda64(value, oa, ref, shapes, P, heads)
    assert bool((want == 0).any()), "the case has no row with every point outside"
    C, S = heads * 32, value.shape[1]
    og, rg = oa.to(DEV), ref.to(DEV)
    fused = torch.full((B, S, 6 * C), float("nan"), dtype=v_dt)
    fused[..., 2 * C:3 * C] = value
    vq = fused.to(DEV)[..., 2 * C:3 * C]
    out = ops.msda(vq, og, rg, shapes, P, heads)
    assert out.dtype == v_dt
    assert_close(out, want, FWD_TOL, f"{case} {dtypes} vector kernel", f16)
    odd = torch.full((B, S, C + 2), float("nan"), dtype=v_dt)
    odd[..., 1:C + 1] = value
    out_s = ops.msda(odd.to(DEV)[..., 1:C + 1], og, rg, shapes, P, heads)
    assert_close(out_s, want, FWD_TOL, f"{case} {dtypes} scalar kernel", f16)
    # the two kernels differ only in the order of the 4*L*P products (fp16 outputs: by at most one rounding)
    a, b = out.cpu().to(F64), out_s.cpu().to(F64)
    bound = 2e-6 * float(want.abs().max()) + (2.0 ** -10 * torch.maximum(a.abs(), b.abs()) if f16 else 0.0)
    assert bool(((a - b).abs() <= bound).all()), f"{case} {dtypes}: scalar and vector kernels differ by {float((a - b).abs().max()):.3e}"
    if dtypes == "f32":
        pair = ops.msda(vq, og, rg, shapes, P, heads, out_pair=True)
        hi, lo = pair.hi.cpu().to(F64), pair.lo.cpu().to(F64)
        assert_close(hi + lo, want, FWD_TOL, f"{case} pair rows hi + lo")
        assert bool((lo.abs() <= 2.0 ** -11 * hi.abs() + 2.0 ** -25).all()), f"{case}: lo is not the fp16 remainder of hi"


# ---- backward --------------------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", list(BWD_CASES))
def test_msda_backward(be, case):
    """MSDAFn forward and backward against fp64 autograd, on boundary-free points (see make_inputs); ref gets no gradient"""
    B, Q, heads, P, shapes, seed = BWD_CASES[case]
    value, oa, ref = make_inputs(B, Q, heads, shapes, P, seed + 100, boundary_free=True)
    dy = torch.randn((B, Q, heads * 32), generator=torch.Generator().manual_seed(seed))
    out64, dv64, doa64 = fwd_bwd64(value, oa, ref, dy, shapes, P, heads)
    vg, og, rg = value.to(DEV).requires_grad_(True), oa.to(DEV).requires_grad_(True), ref.to(DEV).requires_grad_(True)
    y = A.MSDAFn.apply(vg, og, rg, shapes, P, heads)
    y.backward(dy.to(DEV))
    assert rg.grad is None
    assert_close(y, out64, FWD_TOL, f"{case}: out")
    check_grads(vg.grad, og.grad, dv64, doa64, heads, len(shapes), P, case)


@gpu
def test_msda_backward_at_whole_pixel_positions(be):
    """sampling coordinates exactly on whole pixels in fp32 and fp64 (dyadic inputs): the offset gradient is the one of the cell to the right and
    below (floor), as in fp64 autograd of grid_sample; points at ix = -1 and W-1 have one in-map corner and a non-zero offset gradient"""
    B, Q, heads, P = 2, 64, 8, 4
    value, oa, ref = make_dyadic_inputs(B, Q, heads, DYADIC_SHAPES, P, 21)
    dy = torch.randn((B, Q, heads * 32), generator=torch.Generator().manual_seed(22))
    out64, dv64, doa64 = fwd_bwd64(value, oa, ref, dy, DYADIC_SHAPES, P, heads)
    vg, og = value.to(DEV).requires_grad_(True), oa.to(DEV).requires_grad_(True)
    y = A.MSDAFn.apply(vg, og, ref.to(DEV), DYADIC_SHAPES, P, heads)
    y.backward(dy.to(DEV))
    assert_close(y, out64, FWD_TOL, "whole pixels: out")
    check_grads(vg.grad, og.grad, dv64, doa64, heads, len(DYADIC_SHAPES), P, "whole pixels")


@gpu
def test_msda_bwd_abi_accumulates_on_pitched_views_and_doa_is_deterministic(be):
    """fb200_msda_bwd through the backend: value, oa, dout, dvalue and doa as column slices of wider buffers (columns outside the slices of the
    inputs hold NaN, of the outputs known values that must survive), dvalue accumulated onto its prefill, doa bitwise identical across calls"""
    B, Q, heads, P, shapes, seed = CASES["odd"]
    L, C = len(shapes), heads * 32
    n_oa = heads * L * P * 3
    value, oa, ref = make_inputs(B, Q, heads, shapes, P, seed + 200, boundary_free=True)
    S = value.shape[1]
    dy = torch.randn((B, Q, C), generator=torch.Generator().manual_seed(31))
    _, dv64, doa64 = fwd_bwd64(value, oa, ref, dy, shapes, P, heads)
    nan = float("nan")

    def embed(t, width, at, fill):
        buf = torch.full((*t.shape[:-1], width), fill)
        buf[..., at:at + t.shape[-1]] = t
        return buf.to(DEV)

    vb, ob, db = embed(value, 6 * C, C, nan), embed(oa, n_oa + 8, 4, nan), embed(dy, C + 64, 32, nan)
    prefill = torch.randn((B, S, C + 64), generator=torch.Generator().manual_seed(32))
    dvb = prefill.to(DEV, copy=True)
    doab = torch.full((B, Q, n_oa + 12), 7.0, device=DEV)
    args = (vb[..., C:2 * C], ob[..., 4:4 + n_oa], ref.to(DEV), db[..., 32:32 + C], shapes, P, heads, dvb[..., 16:16 + C], doab[..., 8:8 + n_oa])
    be.msda_bwd(*args)
    first = doab.clone()
    got_dv = dvb.cpu().to(F64) - prefill.to(F64)
    assert_close(got_dv[..., 16:16 + C], dv64, 5e-5, "pitched: dvalue - prefill")
    assert torch.equal(dvb.cpu()[..., :16], prefill[..., :16]) and torch.equal(dvb.cpu()[..., 16 + C:], prefill[..., 16 + C:])
    check_grads(got_dv[..., 16:16 + C], first.cpu()[..., 8:8 + n_oa], dv64, doa64, heads, L, P, "pitched")
    assert bool((first[..., :8] == 7).all() and (first[..., 8 + n_oa:] == 7).all())
    be.msda_bwd(*args)   # a second call adds the gradient again and rewrites doa with the same bits
    assert torch.equal(doab, first)
    assert_close(dvb.cpu().to(F64)[..., 16:16 + C] - prefill[..., 16:16 + C].to(F64), 2 * dv64, 5e-5, "pitched: dvalue after two calls - prefill")


# ---- argument checks -----------------------------------------------------------------------------------------------------------------------------------------
def _narrow_pitch(t, pitch):
    """the rows of t read at a pitch smaller than their width: neighbouring rows overlap, and every element stays inside t's storage"""
    return t.as_strided(t.shape, (t.shape[1] * pitch, pitch, 1))


@gpu
def test_msda_argument_checks(be):
    """pitches smaller than the row width and L*P = 33 are rejected on the host, before any launch (the outputs keep their sentinels)"""
    B, Q, heads, P, shapes = 2, 8, 2, 4, [(6, 5), (3, 3)]
    L, C = len(shapes), heads * 32
    value, oa, ref = (t.to(DEV) for t in make_inputs(B, Q, heads, shapes, P, 41))
    dout = torch.randn((B, Q, C), device=DEV)
    dvalue = torch.zeros_like(value)
    doa = torch.full_like(oa, float("nan"))
    out = torch.full((B, Q, C), 5.0, device=DEV)
    n_oa = heads * L * P * 3
    narrow = {"oa_pitch": ("oa", n_oa - 1), "doa_pitch": ("doa", n_oa - 2), "v_pitch": ("value", C - 32), "dv_pitch": ("dvalue", C - 4), "do_pitch": ("do", C - 1)}
    for name, (arg, pitch) in narrow.items():
        args = dict(value=value, oa=oa, ref=ref, do=dout, shapes=shapes, P=P, heads=heads, dvalue=dvalue, doa=doa)
        args[arg] = _narrow_pitch(args[arg], pitch)
        with pytest.raises(RuntimeError, match=f"msda_bwd: {name} \\({pitch}\\)"):
            be.msda_bwd(**args)
    with pytest.raises(RuntimeError, match="msda: oa_pitch"):
        be.msda(value, _narrow_pitch(oa, n_oa - 1), ref, shapes, P, heads, out)
    # pair rows need the vector kernel: a value whose rows are not 16-byte aligned is refused, not sent to the scalar kernel
    vodd = torch.zeros((B, value.shape[1], C + 2), device=DEV)[..., 1:C + 1]
    with pytest.raises(RuntimeError, match="pair output"):
        be.msda(vodd, oa, ref, shapes, P, heads, ops.Pair(torch.full((B, Q, 2 * C), 5.0, dtype=torch.float16, device=DEV)))
    # L*P = 33 > one warp (inputs sized for it)
    shapes33, P33 = [(4, 4), (2, 2), (1, 1)], 11
    v33 = torch.randn((B, 21, C), device=DEV)
    oa33 = torch.randn((B, Q, heads * 33 * 3), device=DEV)
    doa33 = torch.full_like(oa33, float("nan"))
    with pytest.raises(RuntimeError, match="levels\\*points"):
        be.msda(v33, oa33, ref, shapes33, P33, heads, out)
    with pytest.raises(RuntimeError, match="levels\\*points"):
        be.msda_bwd(v33, oa33, ref, dout, shapes33, P33, heads, torch.zeros_like(v33), doa33)
    torch.cuda.synchronize()
    assert bool((dvalue == 0).all() and doa.isnan().all() and (out == 5).all() and doa33.isnan().all())
