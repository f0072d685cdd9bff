"""-m gpu: the residual epilogue of the wgmma conv/linear kernel, bit for bit.

With a ReLU (or no) activation the fused epilogue computes act(v + r) or act(v) + r in fp32, where v = acc * scale + bias is exactly what the same
launch without a residual writes as fp32.  So every residual case here is checked for equality with torch's fp32 arithmetic on that v: a residual
byte read from the wrong ring entry, chunk, row or channel shows up as a mismatch, not as a tolerance question.  The shapes reach every kernel
configuration that loads the residual through the operand ring (fp32-accurate fused split at N = 128 / 64 with 64- and 32-channel k-blocks; fp16
and fp32 output at N = 128 / 64) and the 32-channel fp16 configuration that still loads it into the output staging buffer; they include odd and
even k-block counts, ragged tiles, Cout tails, residuals that are channel slices of wider buffers, and enough tiles that each CTA wraps its ring
many times.  Kept apart from test_gpu_conv_tc.py for the same reason: a barrier-phase bug traps."""
import math

import pytest
import torch

from focoos_b200 import ops
from focoos_b200.engine import _split3_weights
from oracle.ops_ref import RefBackend

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda"
RELU, AFTER = ops.ACT_RELU, 16  # 16: residual added after the activation


def rnd(shape, dtype, seed, s=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * s).to(dtype)


def operands(B, H, W, Cin, Cout, k, seed, dtype):
    x = rnd((B, H, W, Cin), dtype, seed + 1, 3.0 if dtype == torch.float32 else 1.0).to(DEV)
    w = rnd((Cout, k, k, Cin), dtype, seed + 2, 1.0 / math.sqrt(k * k * Cin)).to(DEV)
    sc = (torch.rand(Cout, generator=torch.Generator().manual_seed(seed + 3)) + 0.5).to(DEV)
    bi = rnd((Cout,), torch.float32, seed + 4, 0.2).to(DEV)
    return x, w, sc, bi


def residual_of(shape, dtype, seed, slice_off):
    """a residual tensor; slice_off > 0: channels [slice_off, slice_off + C) of a wider buffer (pitch != C)"""
    C = shape[-1]
    wide = rnd((*shape[:-1], C + 2 * slice_off), dtype, seed, 2.0).to(DEV)
    return wide[..., slice_off:slice_off + C]


def expected(v, r, post):
    return torch.relu(v) + r if post else torch.relu(v + r)


# (B, H, W, Cin, Cout, k): 1x1 with one and three 64-channel k-blocks, 3x3 with 9 / 18; ragged 20x20 / 40x40 / 7x9 maps; Cout tails 96 and 288
SHAPES_K64 = [(2, 20, 20, 64, 256, 1), (2, 40, 40, 192, 256, 1), (2, 20, 20, 64, 96, 3), (2, 40, 40, 128, 288, 3), (3, 7, 9, 64, 128, 3)]
# many tiles per CTA: 1x1 convs / linears over 51,200 - 135,168 rows (each CTA walks its ring dozens of times), and a flat M that is not a multiple of 128
SHAPES_LONG = [(2, 160, 160, 64, 256, 1), (1, 1, 132 * 128 * 8, 64, 128, 1), (1, 1, 1000, 192, 288, 1)]


@pytest.mark.parametrize("post", [False, True])
@pytest.mark.parametrize("out_pair", [True, False])
@pytest.mark.parametrize("B,H,W,Cin,Cout,k", SHAPES_K64 + SHAPES_LONG
                         + [(2, 20, 20, 64, 64, 3), (2, 40, 40, 192, 32, 1), (1, 1, 9600, 64, 64, 1)]       # fused split, N = 64 (Cout 64 and a 32-channel tail)
                         + [(2, 20, 20, 32, 128, 3), (2, 40, 40, 96, 96, 1), (2, 20, 20, 32, 64, 1),         # fused split, 32-channel k-blocks: two ring entries
                            (2, 40, 40, 32, 32, 3), (1, 1, 132 * 128 * 4, 32, 128, 1)])                      # per residual tile (N = 128 and N = 64)
def test_fused_split_residual_bit_exact(B, H, W, Cin, Cout, k, out_pair, post):
    x, w, sc, bi = operands(B, H, W, Cin, Cout, k, Cin + Cout + k, torch.float32)
    xp, w3 = ops.Pair(ops.split_pair(x)), _split3_weights(w)
    pad = (k - 1) // 2
    v = ops.conv2d_pair(xp, w3, sc, bi, pad=pad, act=ops.ACT_NONE, out_pair=False)
    act = RELU | (AFTER if post else 0)
    if out_pair:  # channels [32, 32 + Cout) of a wider pair buffer: the lo planes start Cout + 64 channels after the hi planes, pitch 2 * (Cout + 64)
        rp = ops.Pair(ops.split_pair(rnd((*v.shape[:-1], Cout + 64), torch.float32, Cout + 7, 2.0).to(DEV))).slice(32, 32 + Cout)
        got = ops.conv2d_pair(xp, w3, sc, bi, pad=pad, act=act, residual=rp, out_pair=True)
        e = expected(v, rp.float(), post)
        hi = e.half()
        assert torch.equal(got.hi, hi), "hi plane"
        assert torch.equal(got.lo, (e - hi.float()).half()), "lo plane"
        again = ops.conv2d_pair(xp, w3, sc, bi, pad=pad, act=act, residual=rp, out_pair=True)
        assert torch.equal(again.buf, got.buf)
    else:
        r32 = residual_of(v.shape, torch.float32, Cout + 7, 32)
        got = ops.conv2d_pair(xp, w3, sc, bi, pad=pad, act=act, residual=r32, out_pair=False)
        assert torch.equal(got, expected(v, r32, post))
        assert torch.equal(ops.conv2d_pair(xp, w3, sc, bi, pad=pad, act=act, residual=r32, out_pair=False), got)


@pytest.mark.parametrize("post", [False, True])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("B,H,W,Cin,Cout,k", SHAPES_K64 + SHAPES_LONG
                         + [(2, 20, 20, 64, 64, 3), (2, 40, 40, 192, 64, 1), (1, 1, 9600, 64, 64, 1)]        # N = 64
                         + [(2, 20, 20, 32, 64, 3), (2, 40, 40, 32, 128, 1)])                                 # 32-channel k-blocks: residual via the staging buffer
def test_fp16_operand_residual_bit_exact(B, H, W, Cin, Cout, k, out_dtype, post):
    if out_dtype == torch.float16 and Cout % 64:
        pytest.skip("an fp16 residual is consumed in whole 64-channel chunks: Cout % 64 != 0 takes the SIMT kernel")
    x, w, sc, bi = operands(B, H, W, Cin, Cout, k, Cin + Cout + k, torch.float16)
    pad = (k - 1) // 2
    v = ops.conv2d(x, w, sc, bi, pad=pad, out_dtype=torch.float32, algo=ops.ALGO_TCGEN05)
    r = residual_of(v.shape, out_dtype, Cout + 9, 32 if out_dtype == torch.float32 else 64)
    act = RELU | (AFTER if post else 0)
    got = ops.conv2d(x, w, sc, bi, pad=pad, act=act, residual=r, out_dtype=out_dtype, algo=ops.ALGO_TCGEN05)
    assert torch.equal(got, expected(v, r.float(), post).to(out_dtype))
    assert torch.equal(ops.conv2d(x, w, sc, bi, pad=pad, act=act, residual=r, out_dtype=out_dtype, algo=ops.ALGO_TCGEN05), got)


@pytest.mark.parametrize("act", [ops.ACT_SILU | AFTER, ops.ACT_SILU, ops.ACT_GELU])
@pytest.mark.parametrize("B,H,W,Cin,Cout,k", [(2, 20, 20, 256, 256, 3), (1, 1, 1000, 1024, 256, 1)])
def test_residual_with_silu_and_gelu_against_the_cpu_reference(B, H, W, Cin, Cout, k, act):
    """activations torch does not reproduce bit for bit: the CPU reference within the tolerance of the other tensor-core tests, and a repeat run identical"""
    if (act & 15) == ops.ACT_GELU and k != 1:
        pytest.skip("the GELU epilogue serves the FFN linears")
    x, w, sc, bi = operands(B, H, W, Cin, Cout, k, Cin + k + act, torch.float16)
    pad = (k - 1) // 2
    r = residual_of((B, H, W, Cout), torch.float16, 17, 0)
    ref = torch.empty((B, H, W, Cout), dtype=torch.float16)
    RefBackend().conv2d(x.cpu(), w.cpu(), sc.cpu(), bi.cpu(), 1, pad, act, r.cpu(), ref, 0)
    got = ops.conv2d(x, w, sc, bi, pad=pad, act=act, residual=r, out_dtype=torch.float16, algo=ops.ALGO_TCGEN05)
    a, b = got.float().cpu(), ref.float()
    scale = max(1.0, float(b.abs().max()))
    assert float((a - b).abs().max()) <= 3e-3 * scale
    assert torch.equal(ops.conv2d(x, w, sc, bi, pad=pad, act=act, residual=r, out_dtype=torch.float16, algo=ops.ALGO_TCGEN05), got)
