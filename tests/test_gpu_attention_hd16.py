"""Multi-head attention with 16-channel heads (the encoder of the 128-wide MaskFormer pixel decoders: 8 heads x 16 channels) against a float64
reference written in this file.

Entry points and the kernels they reach at head_dim 16:
- `fb200_attention`, fp32 rows and fp16 rows the tensor cores cannot read (pitch not a multiple of 8 halves, rows not 16-byte aligned):
  `attention_hd16_kernel<T, false>` (K / V resident in shared memory, Lk <= 1164), `attention_hd16_kernel<T, true>` above (256-key chunks).
- `fb200_attention`, aligned fp16 rows: `attention_hd16_mma_kernel<false, false>` (Lk <= 2368), `attention_hd16_mma_kernel<false, true>` above.
- `fb200_attention_split`, fp32 output: `attention_hd16_mma_kernel<true, false>` (self-attention L <= 1088), `attention_hd16_mma_kernel<true, true>` above.

Lengths: the encoder's token counts at 320x416 (130), 800x800 (625), 1024x1024 (1024) and 1080x1920 (2040), each path's resident ceiling and one key
past it, and short / odd tails with Lq != Lk.  q and k are column slices of [B, L, 2C] buffers (row pitch 2C), as the encoder's fused q/k
projection writes them; outputs are written into rows of C + 8.  A profiler check confirms which kernel each case launched.

Bars, as a per-element bound on |got - want|: FWD_TOL = 2e-5 of the output scale, plus the first-order effect of rounding the scores
(2 * D*u*scale * sum_j p_j a_j * range(v), a_j = sum_d |q_d||k_jd|, D = 16, u = 2^-24); fp16 outputs also one fp16 rounding of the output and the fp16
rounding of P in the P.V product: 2^-11 * (|want| + P.|V|)."""
import json
import math
import os
import re
import subprocess
import sys
import time

import pytest
import torch

from focoos_b200 import ops

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
F64 = torch.float64
HD, HEADS = 16, 8
C = HD * HEADS
SCALE = 1 / math.sqrt(HD)
U = 2.0 ** -24
FWD_TOL = 2e-5
NAN = float("nan")

SIMT_CEIL, MMA_CEIL, SPLIT_CEIL = 1164, 2368, 1088


@pytest.fixture()
def be():
    """the CUDA backend (never the CPU reference backend some host-graph tests install)"""
    b = ops._be()
    assert isinstance(b, ops.CudaBackend)
    return b


def _heads(t):
    B, L, _ = t.shape
    return t.to(F64).reshape(B, L, HEADS, HD).transpose(1, 2)


def want_and_bound(q, k, v, f16):
    """(want [B, Lq, C] float64, per-element bound of |got - want|)"""
    Q, K, V = _heads(q), _heads(k), _heads(v)
    P = torch.softmax(Q @ K.transpose(-1, -2) * SCALE, -1)
    want = P @ V
    pa = (P * (Q.abs() @ K.abs().transpose(-1, -2))).sum(-1, keepdim=True)
    rng = (V.amax(2) - V.amin(2))[:, :, None, :]
    bound = FWD_TOL * float(want.abs().max()) + 2 * HD * U * SCALE * pa * rng
    if f16:
        bound = bound + 2.0 ** -11 * (want.abs() + P @ V.abs())
    merge = lambda t: t.transpose(1, 2).reshape(q.shape[0], q.shape[1], C)
    return merge(want), merge(bound)


def make_qkv(B, Lq, Lk, seed, dtype):
    """q / k as the column slices [..., :C] / [..., C:] of [B, L, 2C] buffers (one buffer when Lq == Lk, as the encoder's fused projection writes them);
    v contiguous.  Per (query, head): 70 % unit-scale rows, 20 % rows scaled by 4 (peaked softmax), 10 % q = 0 (uniform)"""
    g = torch.Generator().manual_seed(seed)
    qbuf = torch.randn((B, Lq, 2 * C), generator=g)
    kbuf = qbuf if Lq == Lk else torch.randn((B, Lk, 2 * C), generator=g)
    u = torch.rand((B, Lq, HEADS, 1), generator=g)
    s = torch.where(u < 0.7, 1.0, torch.where(u < 0.9, 4.0, 0.0)).expand(B, Lq, HEADS, HD).reshape(B, Lq, C)
    qbuf[..., :C] *= s
    v = torch.randn((B, Lk, C), generator=g)
    qbuf, kbuf, v = qbuf.to(DEV, dtype), kbuf.to(DEV, dtype), v.to(DEV, dtype)
    return qbuf[..., :C], kbuf[..., C:], v


def _offset_rows(t, extra, off):
    """a copy of t whose rows are C + extra elements apart and start `off` elements into the buffer"""
    B, L, _ = t.shape
    buf = torch.zeros(B * L * (C + extra) + off + C, dtype=t.dtype, device=t.device)
    view = buf[off:off + B * L * (C + extra)].view(B, L, C + extra)[..., :C]
    view.copy_(t)
    return view


PATHS = {   # path -> (dtype, layout, kernel of the resident / streaming variant)
    "f32": (torch.float32, None, r"\battention_hd16_kernel<float, (false|true)>"),
    "f16_simt_pitch": (torch.float16, "pitch", r"\battention_hd16_kernel<__half, (false|true)>"),   # rows C + 4 halves apart
    "f16_simt_off8": (torch.float16, "off8", r"\battention_hd16_kernel<__half, (false|true)>"),     # rows 8 bytes past a 16-byte boundary
    "f16_tc": (torch.float16, None, r"\battention_hd16_mma_kernel<false, (false|true)>"),
    "split_f32": (torch.float32, None, r"\battention_hd16_mma_kernel<true, (false|true)>"),
}
CEIL = {"f32": SIMT_CEIL, "f16_simt_pitch": SIMT_CEIL, "f16_simt_off8": SIMT_CEIL, "f16_tc": MMA_CEIL, "split_f32": SPLIT_CEIL}


def run(be, path, q, k, v):
    dtype, how, _ = PATHS[path]
    if how == "pitch":
        q, k, v = (_offset_rows(t, 4, 0) for t in (q, k, v))
    elif how == "off8":
        q, k, v = (_offset_rows(t, 8, 4) for t in (q, k, v))
    out = torch.full((q.shape[0], q.shape[1], C + 8), NAN, dtype=dtype, device=DEV)[..., :C]   # pitched output rows
    be.attention(q, k, v, out, HEADS, SCALE, path == "split_f32")
    return out.to(F64)


def expected_kernel(path, Lk):
    stream = "true" if Lk > CEIL[path] else "false"
    return PATHS[path][2].replace("(false|true)", stream)


def attention_kernels(prof):
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "attention" in e.name]
    return [e.name for e in sorted(ev, key=lambda e: e.time_range.start)]


SHIPPED = (130, 625, 1024, 2040)
TAILS = [(3, 1, 1), (2, 17, 65), (1, 193, 257), (2, 65, 15), (4, 130, 130)]   # (B, Lq, Lk)


def cases_for(path):
    ceil = CEIL[path]
    c = [(2 if L < 2000 else 1, L, L) for L in SHIPPED] + [(1, ceil, ceil), (2, ceil + 1, ceil + 1)] + TAILS
    return c


@pytest.mark.parametrize("path", list(PATHS))
def test_attention_hd16_vs_float64(be, path):
    """every case of the path against the float64 reference"""
    dtype = PATHS[path][0]
    for n, (B, Lq, Lk) in enumerate(cases_for(path)):
        q, k, v = make_qkv(B, Lq, Lk, 100 + n, dtype)
        got = run(be, path, q, k, v)
        assert bool(torch.isfinite(got).all()), f"{path} B={B} Lq={Lq} Lk={Lk}: non-finite output"
        want, bound = want_and_bound(q, k, v, dtype == torch.float16)
        err = (got - want).abs()
        assert bool((err <= bound).all()), f"{path} B={B} Lq={Lq} Lk={Lk}: max |err| {float(err.max()):.3g}, worst err/bound {float((err / bound).max()):.3g}"


def launched_kernels():
    """[[path, B, Lq, Lk, names of the attention kernels the call launched], ...] from torch.profiler sessions, one per case.  A session can miss a launch
    (the first one especially), so each call runs once before its session and three times inside it."""
    from torch.profiler import ProfilerActivity, profile

    be, res = ops._be(), []
    for path in PATHS:
        for n, (B, Lq, Lk) in enumerate(cases_for(path)):
            q, k, v = make_qkv(B, Lq, Lk, 100 + n, PATHS[path][0])
            run(be, path, q, k, v)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                time.sleep(0.2)  # kernels launched right as a session starts have been seen missing from its trace: start the work 0.2 s in
                for _ in range(3):
                    run(be, path, q, k, v)
                torch.cuda.synchronize()
            res.append([path, B, Lq, Lk, attention_kernels(prof)])
    return res


def test_attention_hd16_dispatch():
    """each case launches the intended kernel: the resident one up to the path's ceiling, the streaming one past it.  The names come from a fresh
    interpreter: in a process where earlier tests ran profiler sessions, a later session has been seen to record no kernels at all."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import json; from tests.test_gpu_attention_hd16 import launched_kernels; print(json.dumps(launched_kernels()))"],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    for path, B, Lq, Lk, names in json.loads(r.stdout.strip().splitlines()[-1]):
        pattern = expected_kernel(path, Lk)
        assert names and all(re.search(pattern, nm) for nm in names), f"{path} B={B} Lq={Lq} Lk={Lk}: expected {pattern}, launched {names}"


@pytest.mark.parametrize("path", ["f32", "f16_tc", "split_f32"])
def test_attention_hd16_batch_rows_independent(be, path):
    """each image of a batch gets exactly the output it gets alone (the encoder's batch invariance)"""
    dtype = PATHS[path][0]
    q, k, v = make_qkv(3, 625, 625, 7, dtype)
    full = run(be, path, q, k, v)
    for b in range(3):
        one = run(be, path, q[b:b + 1], k[b:b + 1], v[b:b + 1])
        assert torch.equal(one[0], full[b])


def test_attention_hd16_argument_checks(be):
    """head_dim outside {16, 32}, pitches below heads*16 and pair output at head_dim 16 are refused on the host, naming the argument, before any
    launch: the output keeps its sentinel"""
    x = torch.randn((2, 16, 2 * C), device=DEV)
    out = torch.full((2, 16, 2 * C), 7.0, device=DEV)
    p, o, st = x.data_ptr(), out.data_ptr(), ops._stream()

    def fwd(hd=HD, heads=HEADS, qp=2 * C):
        be._call("fb200_attention", p, qp, p, 2 * C, p, 2 * C, o, 2 * C, ops.F32, 2, 16, 16, heads, hd, SCALE, st)

    def split(hd=HD, heads=HEADS, qp=2 * C, out_dtype=ops.F32):
        be._call("fb200_attention_split", p, qp, p, 2 * C, p, 2 * C, o, out_dtype, 2 * C, 2, 16, 16, heads, hd, SCALE, st)

    for name, fn in (("attention", fwd), ("attention_split", split)):
        for hd in (0, 8, 24, 64):
            with pytest.raises(RuntimeError, match=rf"\(-1\).*{name}: head_dim must be 16 or 32 \(got {hd}\)"):
                fn(hd=hd, heads=2 * C // max(hd, 1) if hd else 8)
        with pytest.raises(RuntimeError, match=rf"\(-1\).*{name}: q_pitch \(124\) < heads\*16 \(128\)"):
            fn(qp=124)
    with pytest.raises(RuntimeError, match=r"\(-1\).*attention_split: head_dim 16 writes fp32 rows only"):
        split(out_dtype=ops.F16PAIR)
    torch.cuda.synchronize()
    assert bool((out == 7).all())
