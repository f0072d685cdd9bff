"""-m gpu: the wgmma implicit-GEMM conv/linear kernel against the CPU reference (fp32 accumulation of the same
fp16 operands).  Kept in its own file: a descriptor bug would hang or trap, and must not take the SIMT tests down."""
import math

import pytest
import torch

from focoos_b200 import ops
from oracle.ops_ref import RefBackend

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]
REF = RefBackend()
DEV = "cuda"


def rnd(shape, dtype, seed, s=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * s).to(dtype)


def run_case(B, H, W, Cin, Cout, k, stride, act=0, use_res=False, use_scale=True, out_dtype=torch.float16, seed=0, tolerance=3e-3):
    x = rnd((B, H, W, Cin), torch.float16, seed + 1)
    w = rnd((Cout, k, k, Cin), torch.float16, seed + 2, 1.0 / math.sqrt(k * k * Cin))
    sc = (torch.rand(Cout) + 0.5) if use_scale else None
    bi = rnd((Cout,), torch.float32, seed + 3, 0.2)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    res = rnd((B, Ho, Wo, Cout), out_dtype, seed + 4) if use_res else None
    ref = torch.empty((B, Ho, Wo, Cout), dtype=out_dtype)
    REF.conv2d(x, w, sc, bi, stride, pad, act, res, ref, 0)
    out = ops.conv2d(x.to(DEV), w.to(DEV), None if sc is None else sc.to(DEV), bi.to(DEV), stride=stride, pad=pad, act=act,
                     residual=None if res is None else res.to(DEV), out_dtype=out_dtype, algo=ops.ALGO_TCGEN05)
    torch.cuda.synchronize()
    a, b = out.float().cpu(), ref.float()
    err = float((a - b).abs().max())
    scale = max(1.0, float(b.abs().max()))
    assert err <= tolerance * scale, f"tensor-core conv B{B} {H}x{W} {Cin}->{Cout} k{k} s{stride}: max|d|={err:.3e} (scale {scale:.2e}); frac bad={(float(((a-b).abs()>tolerance*scale).float().mean())):.4f}"


@pytest.mark.parametrize("M,K,N", [(128, 64, 64), (256, 128, 128), (1000, 256, 256), (300, 256, 288), (777, 1024, 256), (128, 256, 512), (9600, 256, 1536)])
def test_linear_flat(M, K, N):
    run_case(1, 1, M, K, N, 1, 1, seed=M + K + N)


def test_linear_fp32_out_and_odd_n():
    run_case(1, 1, 500, 256, 368, 1, 1, out_dtype=torch.float32, use_scale=False, tolerance=2e-3)
    run_case(1, 1, 300, 256, 4, 1, 1, out_dtype=torch.float32, use_scale=False, tolerance=2e-3)
    run_case(1, 1, 300, 256, 80, 1, 1, out_dtype=torch.float32, use_scale=False, tolerance=2e-3)


@pytest.mark.parametrize("H,W,Cin,Cout", [(16, 16, 64, 64), (20, 20, 256, 256), (40, 40, 256, 256), (80, 80, 128, 128), (24, 40, 64, 128), (7, 9, 64, 64)])
def test_conv3x3_s1(H, W, Cin, Cout):
    run_case(2, H, W, Cin, Cout, 3, 1, act=1, seed=H + Cin)


@pytest.mark.parametrize("H,W,Cin,Cout", [(40, 40, 128, 128), (16, 24, 64, 64), (80, 80, 256, 256)])
def test_conv3x3_s2(H, W, Cin, Cout):
    run_case(2, H, W, Cin, Cout, 3, 2, act=1, seed=H + Cout)


def test_epilogue_variants():
    run_case(2, 20, 20, 256, 1024, 1, 1, act=1, use_res=True, seed=5)           # bottleneck tail: residual then ReLU
    run_case(2, 20, 20, 256, 256, 3, 1, act=2 | 16, use_res=True, use_scale=False, seed=6)  # CSP tail: SiLU then residual
    run_case(3, 10, 10, 512, 256, 1, 1, act=2, seed=7)
    run_case(1, 1, 400, 256, 1024, 1, 1, act=3, use_scale=False, seed=8)        # GELU FFN


def test_slices_and_batch_stride():
    xb = rnd((2, 20, 20, 512), torch.float16, 50)
    w = rnd((256, 3, 3, 256), torch.float16, 51, 0.02)
    bi = rnd((256,), torch.float32, 52)
    ref = torch.empty((2, 20, 20, 256), dtype=torch.float16)
    REF.conv2d(xb[..., :256], w, None, bi, 1, 1, 2, None, ref, 0)
    xg = xb.to(DEV)
    ob = torch.zeros((2, 20, 20, 512), dtype=torch.float16, device=DEV)
    ops.conv2d(xg[..., :256], w.to(DEV), None, bi.to(DEV), pad=1, act=2, out=ob[..., 256:], algo=ops.ALGO_TCGEN05)
    assert float((ob[..., 256:].float().cpu() - ref.float()).abs().max()) <= 3e-3 * max(1.0, float(ref.abs().max()))
    assert float(ob[..., :256].abs().max()) == 0.0
    w1 = rnd((256, 1, 1, 256), torch.float16, 53, 0.06)
    ref1 = torch.empty((2, 20, 20, 256), dtype=torch.float16)
    REF.conv2d(xb[..., 256:], w1, None, bi, 1, 0, 0, None, ref1, 0)
    mem = torch.zeros((2, 500, 256), dtype=torch.float16, device=DEV)
    ops.conv2d(xg[..., 256:], w1.to(DEV), None, bi.to(DEV), out=mem[:, 50:450].unflatten(1, (20, 20)), algo=ops.ALGO_TCGEN05)
    assert float((mem[:, 50:450].reshape(2, 20, 20, 256).float().cpu() - ref1.float()).abs().max()) <= 3e-3 * max(1.0, float(ref1.abs().max()))
    assert float(mem[:, :50].abs().max()) == 0.0 and float(mem[:, 450:].abs().max()) == 0.0


@pytest.mark.parametrize("H,W,Cin,Cout,k", [(40, 40, 32, 32, 3), (64, 48, 32, 64, 3), (16, 16, 32, 64, 1), (320, 320, 32, 32, 3), (20, 20, 96, 64, 3)])
def test_conv_cin32_swizzle64(H, W, Cin, Cout, k):
    """Cin % 64 != 0 -> BLOCK_K = 32 variant (64-byte rows, SWIZZLE_64B): the ResNet-vd stem convs."""
    run_case(2, H, W, Cin, Cout, k, 1, act=1, seed=H + Cin + Cout)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,res", [(2, 20, 20, 256, 256, 3, 1, False), (1, 1, 1000, 256, 512, 1, 1, True), (2, 40, 40, 128, 128, 3, 2, False),
                                                          (2, 32, 32, 32, 64, 3, 1, False), (1, 1, 300, 1024, 256, 1, 1, True),
                                                          (2, 40, 200, 32, 64, 3, 1, False), (1, 33, 130, 32, 32, 3, 1, False),   # fused split on 32-channel chunks
                                                          (2, 24, 40, 256, 64, 1, 1, False), (2, 40, 40, 64, 64, 3, 1, False),     # fused split, N = 64
                                                          (3, 20, 20, 512, 2048, 1, 1, True), (2, 80, 80, 256, 256, 3, 2, False)])  # pair + residual (2-stage ring), stride-2 pair
def test_split_precision_conv_matches_fp32(B, H, W, Cin, Cout, k, stride, res):
    """precision="fp32_tc": fp32 tensors, three fp16 tensor-core products (hi*hi + hi*lo + lo*hi) -> fp32-level agreement."""
    from focoos_b200.engine import _split3_weights

    x = rnd((B, H, W, Cin), torch.float32, 1, 3.0)
    w = rnd((Cout, k, k, Cin), torch.float32, 2, 1.0 / math.sqrt(k * k * Cin))
    bi, sc = rnd((Cout,), torch.float32, 3, 0.2), torch.rand(Cout) + 0.5
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    r = rnd((B, Ho, Wo, Cout), torch.float32, 4) if res else None
    ref = torch.empty((B, Ho, Wo, Cout), dtype=torch.float32)
    REF.conv2d(x, w, sc, bi, stride, pad, 1, r, ref, 0)
    xp = ops.split_pair(x.to(DEV))
    hi = x.half()
    assert torch.equal(xp.cpu()[..., :Cin], hi) and torch.equal(xp.cpu()[..., Cin:], (x - hi.float()).half())
    out = ops.conv2d_pair(ops.Pair(xp), _split3_weights(w).to(DEV), sc.to(DEV), bi.to(DEV), stride=stride, pad=pad, act=1, residual=None if r is None else r.to(DEV),
                          out_pair=False)
    err = float((out.cpu() - ref).abs().max())
    scale = max(1.0, float(ref.abs().max()))
    assert err <= 2e-5 * scale, f"split-precision conv: max|d|={err:.3e} scale={scale:.2e}"


def test_split_precision_conv_has_no_fp16_output():
    """a split-precision conv writes fp32 or the pair: an fp16 output is refused on the host, before any launch, and fp32 is the default.  ops.conv2d with
    ALGO_TCGEN05_SPLIT3 on the dense [hi|lo] tensor is conv2d_pair with a plain output, bit for bit."""
    from focoos_b200.engine import _split3_weights

    xp = ops.split_pair(rnd((2, 20, 20, 64), torch.float32, 1).to(DEV))
    w3 = _split3_weights(rnd((64, 3, 3, 64), torch.float32, 2, 0.04)).to(DEV)
    with pytest.raises(RuntimeError, match=r"\(-2\).*tensor-core path does not support.*split-precision convs write fp32 or the fp16 pair"):
        ops.conv2d(xp, w3, pad=1, act=ops.ACT_RELU, out_dtype=torch.float16, algo=ops.ALGO_TCGEN05_SPLIT3)
    out = ops.conv2d(xp, w3, pad=1, act=ops.ACT_RELU, algo=ops.ALGO_TCGEN05_SPLIT3)
    assert out.dtype == torch.float32
    assert torch.equal(out, ops.conv2d_pair(ops.Pair(xp), w3, pad=1, act=ops.ACT_RELU, out_pair=False))


def test_conv2d_refuses_the_split_algo_and_per_image_weights_with_a_residual():
    """split-precision products are fb200_conv2d_pair's alone: fb200_conv2d refuses algo 3 (and any other unknown algo); per-image weights take no residual"""
    be = ops._be()
    x, out = torch.zeros((2, 8, 8, 64), dtype=torch.float16, device=DEV), torch.zeros((2, 8, 8, 64), dtype=torch.float16, device=DEV)
    w = torch.zeros((64, 1, 1, 64), dtype=torch.float16, device=DEV)
    for algo in (3, 7):
        with pytest.raises(RuntimeError, match=r"\(-1\).*unknown algo.*fb200_conv2d_pair"):
            be.conv2d(x, w, None, None, 1, 0, ops.ACT_NONE, None, out, algo)
    w5 = torch.zeros((2, 64, 1, 1, 64), dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError, match=r"\(-1\).*per-image weights take no residual"):
        be.conv2d(x, w5, None, None, 1, 0, ops.ACT_NONE, torch.zeros_like(out), out, ops.ALGO_AUTO)
    xp, w35 = ops.Pair(torch.zeros((2, 8, 8, 128), dtype=torch.float16, device=DEV)), torch.zeros((2, 64, 1, 1, 192), dtype=torch.float16, device=DEV)
    out32 = torch.zeros((2, 8, 8, 64), device=DEV)
    with pytest.raises(RuntimeError, match=r"\(-1\).*per-image weights take no residual"):
        be.conv2d_pair(xp, w35, None, None, 1, 0, ops.ACT_NONE, torch.zeros_like(out32), out32)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("B,H,W,C,Q", [(3, 40, 52, 256, 100), (2, 64, 128, 128, 100), (5, 8, 8, 64, 7)])
def test_per_image_weights_product(B, H, W, C, Q, dtype):
    """einsum('bqc,bchw->bqhw') as ONE launch with a per-image weight set (3-D weight tensor map on the tensor-core path)."""
    x = rnd((B, H, W, C), dtype, 1)
    w = rnd((B, Q, 1, 1, C), dtype, 2, 1.0 / math.sqrt(C))
    ref = torch.einsum("bhwc,bqc->bhwq", x.float(), w.float().reshape(B, Q, C))
    Qp = (Q + 7) // 8 * 8
    out = torch.zeros((B, H, W, Qp), dtype=dtype, device=DEV)
    ops.conv2d_per_image(x.to(DEV), w.to(DEV), out=out[..., :Q])
    got = out.cpu().float()
    tol = 3e-3 if dtype == torch.float16 else 1e-4
    scale = max(1.0, float(ref.abs().max()))
    assert float((got[..., :Q] - ref).abs().max()) <= tol * scale
    assert float(got[..., Q:].abs().max()) == 0.0, "padding channels must stay untouched"


@pytest.mark.parametrize("dtype", [torch.float16])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 40, 40, 256, 512), (3, 16, 24, 512, 1024), (1, 80, 80, 64, 128)])
def test_avgpool_folded_into_2x2_stride2_conv(B, H, W, Cin, Cout, dtype):
    """AvgPool2d(2,2) + 1x1 conv == 2x2 stride-2 conv with W/4 on every tap (the vd shortcut, resnet.py:91-102) on the tensor-core stride-2 view."""
    x = rnd((B, H, W, Cin), dtype, 1)
    w1 = rnd((Cout, 1, 1, Cin), dtype, 2, 1.0 / math.sqrt(Cin))
    sc, bi = torch.rand(Cout) + 0.5, rnd((Cout,), torch.float32, 3, 0.2)
    pooled = torch.nn.functional.avg_pool2d(x.float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()
    ref = torch.empty((B, H // 2, W // 2, Cout), dtype=torch.float32)
    REF.conv2d(pooled, w1.float(), sc, bi, 1, 0, 0, None, ref, 0)
    wf = (w1 * 0.25).expand(-1, 2, 2, -1).contiguous()
    out = ops.conv2d(x.to(DEV), wf.to(DEV), sc.to(DEV), bi.to(DEV), stride=2, pad=0, algo=ops.ALGO_TCGEN05)
    scale = max(1.0, float(ref.abs().max()))
    assert float((out.float().cpu() - ref).abs().max()) <= 3e-3 * scale


@pytest.mark.parametrize("M,K,N", [(2 * 8400, 256, 365), (4800, 256, 80), (300, 512, 1000), (129, 64, 7)])
def test_linear_rowmax_without_materialising_the_product(M, K, N):
    """enc_outputs_class.max(-1): row maximum of x @ w.T + b computed in the tensor-core epilogue (atomic max across N tiles)."""
    x = rnd((M, K), torch.float16, 1)
    w = rnd((N, K), torch.float16, 2, 1.0 / math.sqrt(K))
    b = rnd((N,), torch.float32, 3, 2.0) - 3.0  # mostly negative rows: exercises the signed atomic max
    ref = (x.float() @ w.float().t() + b).max(-1).values
    got = ops.linear_rowmax(x.to(DEV), w.to(DEV), b.to(DEV)).cpu()
    assert float((got - ref).abs().max()) <= 1e-4 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("B,H,W,Cout", [(2, 40, 200, 32), (1, 33, 320, 64), (2, 16, 64, 64), (3, 9, 131, 32)])
def test_stem_halo_mode(B, H, W, Cout):
    """32-channel 3x3 stride-1 convs (ResNet-vd conv1_2 / conv1_3): 32-channel chunks with 64-byte swizzled rows, ragged rows and images."""
    x = rnd((B, H, W, 32), torch.float16, 1)
    w = rnd((Cout, 3, 3, 32), torch.float16, 2, 1.0 / math.sqrt(288))
    sc, bi = torch.rand(Cout) + 0.5, rnd((Cout,), torch.float32, 3, 0.2)
    ref = torch.empty((B, H, W, Cout), dtype=torch.float32)
    REF.conv2d(x.float(), w.float(), sc, bi, 1, 1, 1, None, ref, 0)
    out = ops.conv2d(x.to(DEV), w.to(DEV), sc.to(DEV), bi.to(DEV), stride=1, pad=1, act=1, algo=ops.ALGO_TCGEN05)
    err = float((out.float().cpu() - ref).abs().max())
    assert err <= 3e-3 * max(1.0, float(ref.abs().max())), err


# ---- pair-format activations: the conv epilogue writes [hi | lo] fp16 planes, reads pair residuals; pools / resize on pairs -------------------------
def _pair_from(x32):
    return ops.Pair(ops.split_pair(x32.to(DEV)))


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,res", [(2, 20, 20, 256, 256, 3, 1, False), (2, 20, 20, 256, 1024, 1, 1, True), (2, 40, 40, 128, 128, 3, 2, False),
                                                          (2, 40, 200, 32, 64, 3, 1, False), (1, 33, 130, 32, 32, 3, 1, False), (2, 24, 40, 256, 64, 1, 1, True),
                                                          (3, 20, 20, 512, 2048, 1, 1, True), (1, 1, 1000, 256, 512, 1, 1, False), (2, 7, 9, 64, 128, 3, 1, True)])
def test_conv2d_pair_output_and_residual(B, H, W, Cin, Cout, k, stride, res):
    """out = Pair: hi + lo reproduce the fp32 reference conv to split precision; the pair residual is read back as hi + lo"""
    from focoos_b200.engine import _split3_weights
    x = rnd((B, H, W, Cin), torch.float32, 1, 3.0)
    w = rnd((Cout, k, k, Cin), torch.float32, 2, 1.0 / math.sqrt(k * k * Cin))
    bi, sc = rnd((Cout,), torch.float32, 3, 0.2), torch.rand(Cout) + 0.5
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    r = rnd((B, Ho, Wo, Cout), torch.float32, 4) if res else None
    ref = torch.empty((B, Ho, Wo, Cout), dtype=torch.float32)
    REF.conv2d(x, w, sc, bi, stride, pad, 1, r, ref, 0)
    rp = None if r is None else _pair_from(r)
    out = ops.conv2d_pair(_pair_from(x), _split3_weights(w).to(DEV), sc.to(DEV), bi.to(DEV), stride=stride, pad=pad, act=1, residual=rp, out_pair=True)
    torch.cuda.synchronize()
    got = out.float().cpu()
    scale = max(1.0, float(ref.abs().max()))
    assert float((got - ref).abs().max()) <= 2e-5 * scale
    hi = out.hi.float().cpu()
    assert torch.equal(out.hi.cpu(), got.half()) or float((hi - got).abs().max()) <= 1e-3 * scale, "hi plane = fp16 of the value"
    # the same conv with fp32 output and fp32 residual must agree with the pair output to the pair's own resolution
    out32 = ops.conv2d_pair(_pair_from(x), _split3_weights(w).to(DEV), sc.to(DEV), bi.to(DEV), stride=stride, pad=pad, act=1, residual=None if r is None else r.to(DEV), out_pair=False)
    assert float((out32.cpu() - got).abs().max()) <= 4e-6 * scale


def test_conv2d_pair_channel_slices_of_a_wider_pair_buffer():
    """CSP pattern: input = channels [0, C) of a 2C pair buffer, residual = channels [C, 2C), output = a slice of another pair buffer"""
    from focoos_b200.engine import _split3_weights
    C = 128
    y12 = rnd((2, 20, 24, 2 * C), torch.float32, 11, 2.0)
    w = rnd((C, 3, 3, C), torch.float32, 12, 0.03)
    bi = rnd((C,), torch.float32, 13, 0.2)
    ref = torch.empty((2, 20, 24, C), dtype=torch.float32)
    REF.conv2d(y12[..., :C].contiguous(), w, None, bi, 1, 1, 2 | 16, y12[..., C:].contiguous(), ref, 0)
    yp = _pair_from(y12)
    dst = ops.Pair(torch.zeros((2, 20, 24, 4 * C), dtype=torch.float16, device=DEV))
    ops.conv2d_pair(yp.slice(0, C), _split3_weights(w).to(DEV), None, bi.to(DEV), pad=1, act=2 | 16, residual=yp.slice(C, 2 * C), out=dst.slice(C, 2 * C))
    assert float((dst.slice(C, 2 * C).float().cpu() - ref).abs().max()) <= 2e-5 * max(1.0, float(ref.abs().max()))
    assert float(dst.slice(0, C).float().abs().max()) == 0.0, "neighbouring channels untouched"


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_pools_on_pairs_match_the_fp32_operator(mode):
    x = rnd((2, 37, 50, 64), torch.float32, 21, 3.0)
    xp = _pair_from(x)
    if mode == 0:
        got, ref = ops.maxpool3x3s2(xp), torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1)
    elif mode == 1:
        got, ref = ops.avgpool2x2(xp), torch.nn.functional.avg_pool2d(x.permute(0, 3, 1, 2), 2, 2, 0, ceil_mode=True)
    else:
        got, ref = ops.resize_bilinear(xp, (74, 100)), torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), size=(74, 100), mode="bilinear", align_corners=False)
    assert isinstance(got, ops.Pair)
    assert float((got.float().cpu() - ref.permute(0, 2, 3, 1)).abs().max()) <= 3e-6 * 12


def test_stem_conv_pair_output():
    img = torch.randint(0, 256, (2, 64, 96, 3), dtype=torch.uint8)
    w, sc, bi = rnd((32, 3, 3, 3), torch.float32, 31, 0.2), torch.rand(32) + 0.5, rnd((32,), torch.float32, 32, 0.1)
    mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
    a = ops.stem_conv(img.to(DEV), w.to(DEV), sc.to(DEV), bi.to(DEV), mean, std, out_dtype=torch.float32)
    p = ops.stem_conv(img.to(DEV), w.to(DEV), sc.to(DEV), bi.to(DEV), mean, std, out_pair=True)
    assert float((p.float() - a).abs().max()) <= 1e-6 * max(1.0, float(a.abs().max()))


def test_linear_rowmax_pair_matches_fp32():
    """query-selection scores of the fp32-accurate mode: max over the 365 class logits per row, straight from the tensor-core epilogue"""
    from focoos_b200.engine import _split3_weights
    x = rnd((3, 1000, 256), torch.float32, 1, 2.0)
    w = rnd((365, 256), torch.float32, 2, 0.08)
    b = rnd((365,), torch.float32, 3, 0.5)
    ref = (x.reshape(-1, 256).double() @ w.double().t() + b.double()).max(-1).values.float().reshape(3, 1000)
    got = ops.linear_rowmax_pair(ops.Pair(ops.split_pair(x.to(DEV))), _split3_weights(w).to(DEV), b.to(DEV))
    assert float((got.cpu() - ref).abs().max()) <= 2e-5 * float(ref.abs().max())


@pytest.mark.parametrize("out_dtype,Cout,pitch", [(torch.float32, 365, 368), (torch.float32, 81, 96), (torch.float16, 100, 104), (torch.float16, 151, 160)],
                         ids=["f32-365", "f32-81", "f16-100", "f16-151"])
def test_cout_tail_inside_a_16_byte_piece_leaves_the_pitch_padding(out_dtype, Cout, pitch):
    """a Cout whose row ends inside a 16-byte piece (the 365-class head, the 100-query fp16 mask product), written into a slice of a wider buffer: the
    columns past the view keep what they held.  A TMA store clips the channel dimension only to whole 16-byte pieces, so the tensor-core kernel refuses
    such a Cout and AUTO runs it on the CUDA cores; before, the tensor-core store also wrote the columns up to the next 16-byte boundary."""
    x = rnd((1, 1, 300, 256), torch.float16, 11)
    w = rnd((Cout, 1, 1, 256), torch.float16, 12, 1.0 / 16)
    bi = rnd((Cout,), torch.float32, 13, 0.2)
    ref = torch.empty((1, 1, 300, Cout), dtype=out_dtype)
    REF.conv2d(x, w, None, bi, 1, 0, 0, None, ref, 0)
    buf = torch.full((1, 1, 300, pitch), float("nan"), dtype=out_dtype, device=DEV)
    with pytest.raises(RuntimeError, match="tensor-core path does not support"):
        ops.conv2d(x.to(DEV), w.to(DEV), None, bi.to(DEV), out=buf[..., :Cout], algo=ops.ALGO_TCGEN05)
    ops.conv2d(x.to(DEV), w.to(DEV), None, bi.to(DEV), out=buf[..., :Cout])
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[..., Cout:]).all()), "a column past the output view was written"
    got = buf[..., :Cout].float().cpu()
    assert float((got - ref.float()).abs().max()) <= (3e-3 if out_dtype == torch.float16 else 1e-4) * max(1.0, float(ref.abs().max()))


def test_conv2d_pair_refuses_a_cout_tail_inside_a_16_byte_piece():
    """the fp32-accurate conv has no other kernel: a 365-channel fp32 output (1460-byte rows) is refused instead of written to 368 columns; the padded
    368-row head the DETR pair flow packs writes its whole view"""
    from focoos_b200.engine import _split3_weights

    x = rnd((1, 1, 300, 256), torch.float32, 21).to(DEV)
    w = rnd((368, 1, 1, 256), torch.float32, 22, 1.0 / 16).to(DEV)
    w[365:] = 0
    buf = torch.full((1, 1, 300, 368), float("nan"), dtype=torch.float32, device=DEV)
    with pytest.raises(RuntimeError, match="tensor-core path does not support"):
        ops.conv2d_pair(ops.to_pair(x), _split3_weights(w[:365]), out=buf[..., :365], out_pair=False)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf).all())
    ops.conv2d_pair(ops.to_pair(x), _split3_weights(w), out=buf, out_pair=False)
    ref = (x.double().reshape(300, 256) @ w.double().reshape(368, 256).t()).reshape(1, 1, 300, 368)
    assert float((buf.double() - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))
    assert float(buf[..., 365:].abs().max()) == 0.0
