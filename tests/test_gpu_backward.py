"""-m gpu: every backward / training-mode kernel (through the C-ABI, via focoos_b200.autograd_ops) against torch CPU autograd of
the torch op the reference calls at that site.  fp32; tolerance = fp32 reassociation relative to the gradient's scale."""
import math

import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import autograd_ops as A
from focoos_b200 import ops

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda"


def rnd(shape, seed, s=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * s


def close(got, ref, what, tol=2e-5):
    got, ref = got.detach().float().cpu(), ref.detach().float()
    scale = max(1e-6, float(ref.abs().max()))
    err = float((got - ref).abs().max())
    assert err <= tol * scale, f"{what}: max|d|={err:.3e} scale={scale:.3e}"


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def leaf(t, dev=None):
    return (t.to(dev) if dev else t.clone()).requires_grad_(True)


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,bias", [(2, 13, 17, 32, 64, 3, 1, False), (2, 16, 20, 64, 32, 3, 2, True), (3, 9, 9, 96, 64, 1, 1, True),
                                                          (2, 15, 15, 32, 32, 3, 2, False), (2, 32, 32, 3, 32, 3, 2, False), (1, 1, 300, 256, 64, 1, 1, True)])
def test_conv2d_grads(B, H, W, Cin, Cout, k, stride, bias, precision):
    x, w = rnd((B, H, W, Cin), 1), rnd((Cout, Cin, k, k), 2, 1 / math.sqrt(Cin * k * k))
    b = rnd((Cout,), 3) if bias else None
    pad = (k - 1) // 2
    xr, wr = leaf(x), leaf(w)
    br = leaf(b) if bias else None
    yr = nhwc(F.conv2d(nchw(xr), wr, br, stride, pad))
    dy = rnd(tuple(yr.shape), 4)
    yr.backward(dy)
    xg, wg = leaf(x, DEV), leaf(w, DEV)
    bg = leaf(b, DEV) if bias else None
    yg = A.conv2d(xg, wg, bg, stride, pad, precision)
    yg.backward(dy.to(DEV))
    tol = 2e-5 if precision == "fp32" else 5e-5
    close(yg, yr, "conv fwd", tol)
    close(xg.grad, xr.grad, "conv dx", tol)
    close(wg.grad, wr.grad, "conv dw", tol)
    if bias:
        close(bg.grad, br.grad, "conv db", tol)


@pytest.mark.parametrize("act,res", [(ops.ACT_NONE, False), (ops.ACT_RELU, False), (ops.ACT_RELU, True), (ops.ACT_SILU, False), (ops.ACT_NONE, True)])
def test_batchnorm_train_grads(act, res):
    B, H, W, C = 3, 11, 7, 64
    x, r = rnd((B, H, W, C), 1, 2.0) + 0.5, rnd((B, H, W, C), 2)
    g, bt = rnd((C,), 3).abs() + 0.5, rnd((C,), 4)
    rm, rv = rnd((C,), 5) * 0.1, rnd((C,), 6).abs() + 0.5
    fa = {ops.ACT_NONE: lambda t: t, ops.ACT_RELU: F.relu, ops.ACT_SILU: F.silu}[act]
    xr, rr, gr, br = leaf(x), leaf(r), leaf(g), leaf(bt)
    rmr, rvr = rm.clone(), rv.clone()
    z = nhwc(F.batch_norm(nchw(xr), rmr, rvr, gr, br, training=True, momentum=0.1, eps=1e-5))
    yr = fa(z + rr if res else z)
    dy = rnd(tuple(yr.shape), 7)
    yr.backward(dy)
    xg, rg, gg, bg = leaf(x, DEV), leaf(r, DEV), leaf(g, DEV), leaf(bt, DEV)
    rmg, rvg = rm.to(DEV), rv.to(DEV)
    yg = A.BatchNormTrainFn.apply(xg, gg, bg, rmg, rvg, rg if res else None, act, 1e-5, 0.1)
    yg.backward(dy.to(DEV))
    close(yg, yr, "bn fwd")
    close(rmg, rmr, "running_mean", 1e-6)
    close(rvg, rvr, "running_var", 1e-6)
    close(xg.grad, xr.grad, "bn dx", 5e-5)
    close(gg.grad, gr.grad, "bn dgamma", 5e-5)
    close(bg.grad, br.grad, "bn dbeta", 5e-5)
    if res:
        close(rg.grad, rr.grad, "bn dres")


@pytest.mark.parametrize("R,C", [(102400, 256), (4800, 365)])
def test_colsum_at_fine_tune_rows(R, C):
    """bias gradients of Conv2dFn / LinearFn at fine-tune row counts, against an fp64 column sum.  R = 102,400 at C = 256 runs col_partial4's
    unrolled four-row loop (R > 3 * 264 * 8) and its tail; 365 (the class head) is not a width the vector kernel takes, so the scalar kernel runs.
    Zero-mean data: a dropped or doubled row moves a column sum by O(1) against a scale of O(sqrt(R)), far above the bar."""
    x = rnd((R, C), 1)
    ref = x.double().sum(0)
    xg = x.to(DEV)
    out, again = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    ops._be().colsum(xg, out)
    ops._be().colsum(xg, again)
    close(out, ref, "colsum", 2e-5)
    assert torch.equal(out, again), "colsum is not bitwise reproducible"


@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("M", [16 * 300, 16 * 400])
def test_layernorm_grads_at_fine_tune_rows(M, res):
    """LayerNormFn backward at the decoder (bs 16 x 300 queries) and AIFI (bs 16 x 20 x 20) row counts, against fp64 autograd: the grid is capped
    at 264 blocks of 8 warps, so each warp walks several rows and the per-block parameter-gradient partials sum over them"""
    C = 256
    x, r = rnd((M, C), 1), rnd((M, C), 2)
    g, b = rnd((C,), 3).abs() + 0.5, rnd((C,), 4)
    xr, rr, gr, br = (t.double().requires_grad_(True) for t in (x, r, g, b))
    yr = F.layer_norm(xr + rr if res else xr, (C,), gr, br, 1e-5)
    dy = rnd((M, C), 5)
    yr.backward(dy.double())
    xg, rg, gg, bg = leaf(x, DEV), leaf(r, DEV), leaf(g, DEV), leaf(b, DEV)
    yg = A.LayerNormFn.apply(xg, rg if res else None, gg, bg, 1e-5)
    yg.backward(dy.to(DEV))
    close(yg, yr, "ln fwd")
    close(xg.grad, xr.grad, "ln dx")
    if res:
        close(rg.grad, rr.grad, "ln dres")
    close(gg.grad, gr.grad, "ln dgamma")
    close(bg.grad, br.grad, "ln dbeta")


def test_layernorm_linear_addact_grads():
    M, C, N = 2 * 37, 256, 96
    x, r = rnd((2, 37, C), 1), rnd((2, 37, C), 2)
    g, b = rnd((C,), 3).abs() + 0.5, rnd((C,), 4)
    xr, rr, gr, br = leaf(x), leaf(r), leaf(g), leaf(b)
    yr = F.layer_norm(xr + rr, (C,), gr, br, 1e-5)
    dy = rnd(tuple(yr.shape), 5)
    yr.backward(dy)
    xg, rg, gg, bg = leaf(x, DEV), leaf(r, DEV), leaf(g, DEV), leaf(b, DEV)
    yg = A.LayerNormFn.apply(xg, rg, gg, bg, 1e-5)
    yg.backward(dy.to(DEV))
    close(yg, yr, "ln fwd")
    close(xg.grad, xr.grad, "ln dx")
    close(rg.grad, rr.grad, "ln dres")
    close(gg.grad, gr.grad, "ln dgamma")
    close(bg.grad, br.grad, "ln dbeta")
    for act, precision in ((ops.ACT_NONE, "fp32"), (ops.ACT_RELU, "fp32"), (ops.ACT_RELU, "fp32_tc")):
        w, bb = rnd((N, C), 6, 1 / 16), rnd((N,), 7)
        xr, wr, br = leaf(x), leaf(w), leaf(bb)
        yr = F.linear(xr, wr, br)
        yr = F.relu(yr) if act == ops.ACT_RELU else yr
        dy = rnd(tuple(yr.shape), 8)
        yr.backward(dy)
        xg, wg, bg = leaf(x, DEV), leaf(w, DEV), leaf(bb, DEV)
        yg = A.linear(xg, wg, bg, act, precision)
        yg.backward(dy.to(DEV))
        tol = 2e-5 if precision == "fp32" else 5e-5
        close(yg, yr, "linear fwd", tol)
        close(xg.grad, xr.grad, "linear dx", tol)
        close(wg.grad, wr.grad, "linear dw", tol)
        close(bg.grad, br.grad, "linear db", tol)
    for act, fa in ((ops.ACT_SILU, F.silu), (ops.ACT_GELU, F.gelu), (ops.ACT_NONE, lambda t: t)):
        ar, br = leaf(x), leaf(r)
        yr = fa(ar + br)
        dy = rnd(tuple(yr.shape), 9)
        yr.backward(dy)
        ag, bg = leaf(x, DEV), leaf(r, DEV)
        yg = A.AddActFn.apply(ag, bg, act)
        yg.backward(dy.to(DEV))
        close(yg, yr, "addact fwd")
        close(ag.grad, ar.grad, "addact da")
        close(bg.grad, br.grad, "addact db")


@pytest.mark.parametrize("H,W", [(16, 16), (15, 21), (7, 9)])
def test_pool_and_resize_grads(H, W):
    B, C = 2, 32
    x = rnd((B, H, W, C), 1)
    for name, fg, fr in (("maxpool", A.MaxPoolFn.apply, lambda t: F.max_pool2d(t, 3, 2, 1)),
                         ("avgpool", A.AvgPoolFn.apply, lambda t: F.avg_pool2d(t, 2, 2, 0, ceil_mode=True)),
                         ("up2", lambda t: A.ResizeFn.apply(t, (2 * H, 2 * W)), lambda t: F.interpolate(t, size=(2 * H, 2 * W), mode="bilinear", align_corners=False)),
                         ("down", lambda t: A.ResizeFn.apply(t, ((H + 1) // 2, (W + 1) // 2)), lambda t: F.interpolate(t, size=((H + 1) // 2, (W + 1) // 2), mode="bilinear", align_corners=False))):
        xr = leaf(x)
        yr = nhwc(fr(nchw(xr)))
        dy = rnd(tuple(yr.shape), 2)
        yr.backward(dy)
        xg = leaf(x, DEV)
        yg = fg(xg)
        yg.backward(dy.to(DEV))
        close(yg, yr, name + " fwd")
        close(xg.grad, xr.grad, name + " dx")


@pytest.mark.parametrize("B,Lq,Lk,heads", [(2, 37, 37, 2), (1, 300, 300, 8), (2, 400, 400, 8), (2, 50, 80, 4)])
def test_attention_grads(B, Lq, Lk, heads):
    C = heads * 32
    q, k, v = rnd((B, Lq, C), 1), rnd((B, Lk, C), 2), rnd((B, Lk, C), 3)
    scale = 1 / math.sqrt(32)

    def core(q, k, v):
        qh, kh, vh = (t.reshape(B, -1, heads, 32).transpose(1, 2) for t in (q, k, v))
        return (torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh).transpose(1, 2).reshape(B, Lq, C)

    qr, kr, vr = leaf(q), leaf(k), leaf(v)
    yr = core(qr, kr, vr)
    dy = rnd(tuple(yr.shape), 4)
    yr.backward(dy)
    qg, kg, vg = leaf(q, DEV), leaf(k, DEV), leaf(v, DEV)
    yg = A.AttentionFn.apply(qg, kg, vg, heads, scale)
    yg.backward(dy.to(DEV))
    close(yg, yr, "attn fwd")
    close(qg.grad, qr.grad, "attn dq", 5e-5)
    close(kg.grad, kr.grad, "attn dk", 5e-5)
    close(vg.grad, vr.grad, "attn dv", 5e-5)


def test_msda_grads():
    from oracle.ops_ref import RefBackend

    B, Q, heads, P = 2, 60, 8, 4
    shapes = [(5, 7), (10, 14), (20, 28)]
    S, L = sum(h * w for h, w in shapes), len(shapes)
    value, oa = rnd((B, S, heads * 32), 1), rnd((B, Q, heads * L * P * 3), 2, 1.5)
    g = torch.Generator().manual_seed(3)
    ref = torch.cat([0.1 + 0.8 * torch.rand((B, Q, 2), generator=g), 0.05 + 0.5 * torch.rand((B, Q, 2), generator=g)], -1)
    dy = rnd((B, Q, heads * 32), 4)
    rb = RefBackend()
    out_ref = torch.empty((B, Q, heads * 32))
    rb.msda(value, oa, ref, shapes, P, heads, out_ref)
    dv_ref, doa_ref = torch.zeros_like(value), torch.empty_like(oa)
    rb.msda_bwd(value, oa, ref, dy, shapes, P, heads, dv_ref, doa_ref)
    vg, og = leaf(value, DEV), leaf(oa, DEV)
    yg = A.MSDAFn.apply(vg, og, ref.to(DEV), shapes, P, heads)
    yg.backward(dy.to(DEV))
    close(yg, out_ref, "msda fwd")
    close(vg.grad, dv_ref, "msda dvalue", 5e-5)
    close(og.grad, doa_ref, "msda doa", 5e-5)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k", [(2, 40, 40, 256, 256, 3), (2, 20, 20, 512, 128, 1), (1, 1, 600, 256, 1024, 1), (2, 16, 24, 64, 64, 3),
                                               (2, 20, 20, 96, 200, 3), (2, 23, 37, 128, 64, 3), (1, 1, 2400, 256, 80, 1), (4, 80, 80, 64, 256, 1),
                                               (2, 96, 96, 32, 32, 3), (2, 96, 96, 32, 64, 3)])
def test_weight_gradient_on_tensor_cores(B, H, W, Cin, Cout, k):
    """wgmma MN-major split-precision weight gradient vs torch's conv2d_weight in fp64 (and it must actually take the tensor-core path).
    The 32-channel stem convs (conv1_2: 32 -> 32, conv1_3: 32 -> 64) fill only half of a 64-channel TMA box with the operand's hi (or lo) plane."""
    x, dy = rnd((B, H, W, Cin), 1), rnd((B, H, W, Cout), 2)
    pad = (k - 1) // 2
    ref = torch.nn.grad.conv2d_weight(nchw(x).double().contiguous(), (Cout, Cin, k, k), nchw(dy).double().contiguous(), stride=1, padding=pad).permute(0, 2, 3, 1)
    be = ops._be()
    assert be.conv_wgrad_tc_supported(tuple(x.shape), tuple(dy.shape), k, k, 1, pad)
    got = A.weight_grad(x.to(DEV), dy.to(DEV), k, k, 1, pad, "fp32_tc")
    close(got, ref.float(), "wgrad tc", 2e-5)
    simt = A.weight_grad(x.to(DEV), dy.to(DEV), k, k, 1, pad, "fp32")
    close(simt, ref.float(), "wgrad simt", 2e-5)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 40, 40, 128, 128), (2, 31, 45, 64, 256), (4, 80, 80, 256, 256)])
def test_stride2_weight_gradient_on_tensor_cores(B, H, W, Cin, Cout):
    """3x3 stride-2 convs: the X operand is gathered by a TMA map that traverses every second pixel (element strides 2)."""
    k, pad = 3, 1
    Ho, Wo = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    x, dy = rnd((B, H, W, Cin), 1), rnd((B, Ho, Wo, Cout), 2)
    ref = torch.nn.grad.conv2d_weight(nchw(x).double().contiguous(), (Cout, Cin, k, k), nchw(dy).double().contiguous(), stride=2, padding=pad).permute(0, 2, 3, 1)
    assert ops._be().conv_wgrad_tc_supported(tuple(x.shape), tuple(dy.shape), k, k, 2, pad)
    got = A.weight_grad(x.to(DEV), dy.to(DEV), k, k, 2, pad, "fp32_tc")
    close(got, ref.float(), "wgrad tc stride 2", 2e-5)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride", [(2, 40, 40, 256, 256, 3, 1), (1, 1, 600, 256, 1024, 1, 1), (2, 23, 37, 128, 64, 3, 1), (2, 31, 45, 64, 256, 3, 2),
                                                      (2, 96, 96, 32, 32, 3, 1), (2, 96, 96, 32, 64, 3, 1)])
def test_weight_gradient_single_product(B, H, W, Cin, Cout, k, stride):
    """"amp" training precision: ONE tensor-core product on fp16-rounded operands (fb200_conv_wgrad_tc_f16), fp32 accumulation: exact (to fp32 summation order)
    for operands that ARE fp16 values, and within the fp16 operand rounding (2^-11 relative per element) of the fp32 gradient otherwise."""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x, dy = rnd((B, H, W, Cin), 1), rnd((B, Ho, Wo, Cout), 2)
    xh, dyh = x.half().float(), dy.half().float()
    ref = torch.nn.grad.conv2d_weight(nchw(xh).double().contiguous(), (Cout, Cin, k, k), nchw(dyh).double().contiguous(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    assert ops._be().conv_wgrad_tc_supported(tuple(x.shape), tuple(dy.shape), k, k, stride, pad)
    got = A.weight_grad(x.to(DEV), dy.to(DEV), k, k, stride, pad, "amp")
    close(got, ref.float(), "wgrad amp (fp16-rounded operands)", 2e-5)
    full = torch.nn.grad.conv2d_weight(nchw(x).double().contiguous(), (Cout, Cin, k, k), nchw(dy).double().contiguous(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    rel = float((got.cpu().double() - full).norm() / full.norm())
    assert rel < 1e-3, rel


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride", [(2, 40, 40, 64, 128, 3, 1), (2, 40, 40, 128, 128, 3, 2), (2, 20, 20, 256, 64, 1, 1)])
def test_conv2d_grads_amp(B, H, W, Cin, Cout, k, stride):
    """Conv2dFn in the "amp" precision: forward, data gradient and weight gradient are single fp16 products with fp32 accumulation - compared with torch fp64 on
    the fp16-rounded operands (forward / dw) and with the fp32 result at the fp16-rounding tolerance (dx: the weights AND dy are rounded)."""
    pad = (k - 1) // 2
    x, w = rnd((B, H, W, Cin), 1), rnd((Cout, Cin, k, k), 2, 0.05)
    xr, wr = leaf(x.half().float()), leaf(w.half().float())
    yr = nhwc(F.conv2d(nchw(xr), wr, None, stride, pad))
    dy = rnd(tuple(yr.shape), 4).half().float()
    yr.backward(dy)
    xg, wg = leaf(x, DEV), leaf(w, DEV)
    yg = A.conv2d(xg, wg, None, stride, pad, "amp")
    yg.backward(dy.to(DEV))
    close(yg, yr, "amp fwd", 2e-5)
    close(wg.grad, wr.grad, "amp dw", 2e-5)
    close(xg.grad, xr.grad, "amp dx", 2e-5)


def test_stem_weight_gradient_kernel():
    """3x3 stride-2 conv on the 3-channel image (conv1_1): dedicated CUDA-core kernel (8x16 dY tile + input halo in shared memory)."""
    B, H, W, Cin, Cout = 2, 70, 100, 3, 32
    x, w = rnd((B, H, W, Cin), 1), rnd((Cout, Cin, 3, 3), 2, 0.2)
    xr, wr = leaf(x), leaf(w)
    yr = nhwc(F.conv2d(nchw(xr), wr, None, 2, 1))
    dy = rnd(tuple(yr.shape), 4)
    yr.backward(dy)
    xg, wg = leaf(x, DEV), leaf(w, DEV)
    yg = A.conv2d(xg, wg, None, 2, 1, "fp32_tc")
    yg.backward(dy.to(DEV))
    close(yg, yr, "stem fwd")
    close(wg.grad, wr.grad, "stem dw")
    close(xg.grad, xr.grad, "stem dx")


@pytest.mark.parametrize("kernel", ["split", "f16"])
@pytest.mark.parametrize("signs", ["random", "same"])
@pytest.mark.parametrize("B,H,W,Cin,Cout,k", [(1, 1, 900, 256, 80, 1), (1, 1, 4800, 256, 1024, 1), (16, 320, 320, 32, 64, 3)])
def test_weight_gradient_long_same_sign_sums(B, H, W, Cin, Cout, k, signs, kernel):
    """the tensor-core weight gradients at the fine-tune step's longest sums (the decoder linears over 300 * B rows; conv1_3 over 16 x 320 x 320
    pixels, ~30 pixel splits of 53k pixels each) against fp64 of the operands they received, at the bars of tests/conv_launch_check.py.  Operands of one
    sign (|x|, |dy|) make every product of a sum the same sign, as the correlated activations and gradients of a training step do: an accumulator whose
    additions do not round to nearest then drifts in proportion to the number of additions into it (5x the per-launch bar over the 900-row linears and
    2.7x the per-element bar over conv1_3 before each 64-pixel chunk got an accumulator of its own)."""
    from tests.conv_launch_check import CheckingBackend

    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn((B, H, W, Cin), generator=g, device=DEV)
    dy = torch.randn((B, H, W, Cout), generator=g, device=DEV) * 0.05
    if signs == "same":
        x, dy = x.abs(), dy.abs()
    pad = (k - 1) // 2
    assert ops._be().conv_wgrad_tc_supported(tuple(x.shape), tuple(dy.shape), k, k, 1, pad)
    chk = CheckingBackend(ops.CudaBackend(), f"wgrad {kernel} {signs}")
    dw = torch.empty((Cout, k, k, Cin), dtype=torch.float32, device=DEV)
    if kernel == "f16":
        chk.conv_wgrad_tc_f16(x.half(), dy.half(), k, k, 1, pad, dw)
    else:
        chk.conv_wgrad_tc(ops.split_pair(x), ops.split_pair(dy), k, k, 1, pad, dw)
    chk.raise_failures()
