"""-m gpu: the fp32-accurate (fused-split) products of conv_tc_kernel, one launch per kernel configuration, against fp64.

At N = 128 the fused-split convs load A_hi and A_lo of each 16-channel step from the swizzled ring tile with ldmatrix and issue hi x W_hi, hi x W_lo and
lo x W_hi with A in registers; a wrong fragment row, column or swizzle phase shows up here as an error far above the split-precision bar.  The N = 64
configurations keep A in shared memory and are held to the same bar next to them.  The cases reach N = 128 and N = 64 tiles on 64-channel (128-byte swizzle)
and 32-channel (64-byte swizzle) k-blocks.  Between them they cover a pair residual, a 3x3 stride-2 conv on an odd map, pair output, odd and even k-block
counts and ragged tiles, and one case long enough that every CTA walks its ring and its fragment buffers over many tiles."""
import math

import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import ops
from focoos_b200.engine import _split3_weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda"


def make(B, H, W, Cin, Cout, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g) * 3.0
    w = torch.randn(Cout, k, k, Cin, generator=g) / math.sqrt(k * k * Cin)
    sc, bi = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g) * 0.2
    return x, w, sc, bi


def ref64(x, w, sc, bi, stride, pad, residual):
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), stride=stride, padding=pad).permute(0, 2, 3, 1)
    y = y * sc.double() + bi.double()
    if residual is not None:
        y = y + residual.double()
    return torch.relu(y)


# (B, H, W, Cin, Cout, k, stride, residual, out_pair)
CASES = {
    "N128-K64-3x3-res-pair": (2, 20, 24, 128, 256, 3, 1, True, True),
    "N128-K64-3x3s2-odd": (2, 45, 61, 64, 128, 3, 2, False, True),
    "N128-K64-1x1-long": (4, 80, 80, 64, 128, 1, 1, True, False),
    "N64-K64-3x3-res-pair": (2, 33, 41, 64, 64, 3, 1, True, True),
    "N64-K64-3x3s2-odd": (2, 23, 31, 128, 64, 3, 2, False, False),
    "N128-K32-3x3-res-pair": (2, 20, 20, 96, 128, 3, 1, True, True),
    "N128-K32-3x3s2-odd": (2, 45, 61, 32, 128, 3, 2, False, True),
    "N64-K32-3x3-pair": (2, 40, 56, 96, 64, 3, 1, False, True),
    "N64-K32-1x1-res": (2, 40, 40, 32, 64, 1, 1, True, False),
}


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,res,out_pair", list(CASES.values()), ids=list(CASES))
def test_fused_split_register_a_matches_fp64(B, H, W, Cin, Cout, k, stride, res, out_pair):
    x, w, sc, bi = make(B, H, W, Cin, Cout, k, B + H + W + Cin + Cout + k + stride)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    r = torch.randn(B, Ho, Wo, Cout, generator=torch.Generator().manual_seed(Cout + 7)) * 2.0 if res else None
    # a pair output takes a pair residual, an fp32 output an fp32 one; the reference adds what the kernel reads
    rd = None if r is None else (ops.to_pair(r.to(DEV)) if out_pair else r.to(DEV))
    r_seen = None if r is None else (rd.float().cpu() if out_pair else r)
    run = lambda: ops.conv2d_pair(ops.to_pair(x.to(DEV)), _split3_weights(w).to(DEV), sc.to(DEV), bi.to(DEV), stride=stride, pad=pad, act=ops.ACT_RELU,
                                  residual=rd, out_pair=out_pair)
    y = run()
    got = y.float() if out_pair else y
    ref = ref64(x, w, sc, bi, stride, pad, r_seen)
    err = float((got.double().cpu() - ref).abs().max())
    scale = max(1.0, float(ref.abs().max()))
    assert err <= 2e-5 * scale, f"max|d|={err:.3e} scale={scale:.2e}"  # the split-precision bar of test_split_precision_conv_matches_fp32
    again = run()
    assert torch.equal(again.buf if out_pair else again, y.buf if out_pair else y), "a repeat launch gives other bits"
