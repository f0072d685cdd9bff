"""The small-channel fp32-accurate 3x3 convs against fp64: the five shipped ResNet-vd shapes (conv1_2 and conv1_3 run on conv_tc_smallc_kernel, with
resident weights and one input patch per output tile; the 64-channel res2 branch2b stays on the general kernel) and ragged maps, with pair and fp32 output,
channel-sliced pair input and batch invariance; and the dispatch boundary between the two kernels."""
import json
import os
import subprocess
import sys
import time

import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import ops
from focoos_b200.engine import _split3_weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]
DEV = "cuda"


def make(B, H, W, Cin, Cout, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, H, W, Cin, generator=g) * 3.0
    w = torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5
    sc, bi = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g) * 0.2
    return x, w, sc, bi


def ref64(x, w, sc, bi, residual=None):
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    y = y * sc.double() + bi.double()
    if residual is not None:
        y = y + residual.double()
    return torch.relu(y)


def check(got, ref):
    err = float((got.double().cpu() - ref).abs().max())
    scale = max(1.0, float(ref.abs().max()))
    assert err <= 2e-5 * scale, f"max|d|={err:.3e} scale={scale:.2e}"  # the split-precision bar of test_split_precision_conv_matches_fp32


def conv(xp, w, sc, bi, out_pair, out=None):
    return ops.conv2d_pair(xp, _split3_weights(w).to(DEV), sc.to(DEV), bi.to(DEV), pad=1, act=ops.ACT_RELU, out=out, out_pair=out_pair)


def as_float(y):
    return y.float() if isinstance(y, ops.Pair) else y


@pytest.mark.parametrize("out_pair", [True, False])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 320, 320, 32, 32), (2, 320, 320, 32, 64), (2, 160, 160, 64, 64),   # conv1_2, conv1_3, res2 branch2b
                                            (3, 7, 9, 32, 32), (2, 33, 41, 32, 64), (1, 321, 17, 32, 64), (2, 33, 41, 64, 64)])
def test_small_channel_conv_matches_fp64(B, H, W, Cin, Cout, out_pair):
    x, w, sc, bi = make(B, H, W, Cin, Cout, H + W + Cin + Cout)
    y = conv(ops.to_pair(x.to(DEV)), w, sc, bi, out_pair)
    check(as_float(y), ref64(x, w, sc, bi))


@pytest.mark.parametrize("Cout", [32, 64])
def test_channel_slice_of_a_wider_pair_buffer(Cout):
    """input = channels [32, 64) of a 96-channel pair buffer (lo plane 96 channels after hi, pixel pitch 192); output = a channel slice too"""
    B, H, W, Cin = 2, 40, 56, 32
    x, w, sc, bi = make(B, H, W, Cin, Cout, 7 + Cout)
    wide = torch.rand(B, H, W, 96) * 3.0
    wide[..., 32:64] = x
    xp = ops.to_pair(wide.to(DEV)).slice(32, 64)
    assert xp.lo_off != xp.C and xp.buf.stride(2) > 2 * xp.C
    obuf = ops.Pair.empty((B, H, W, Cout + 64), DEV)
    obuf.buf.zero_()
    y = conv(xp, w, sc, bi, True, out=obuf.slice(32, 32 + Cout))
    check(y.float(), ref64(x, w, sc, bi))
    assert float(obuf.slice(0, 32).float().abs().max()) == 0.0 and float(obuf.slice(32 + Cout, 64 + Cout).float().abs().max()) == 0.0


@pytest.mark.parametrize("Cout", [32, 64])
def test_batch_invariance(Cout):
    """every image of a batch gets the same bits as when it runs alone"""
    B, H, W, Cin = 3, 45, 70, 32
    x, w, sc, bi = make(B, H, W, Cin, Cout, 11 + Cout)
    xp = ops.to_pair(x.to(DEV))
    full = conv(xp, w, sc, bi, True).buf
    for i in range(B):
        one = conv(ops.to_pair(x[i:i + 1].to(DEV)), w, sc, bi, True).buf
        assert torch.equal(full[i:i + 1], one)


def kernels_run(fn):
    """names of the conv_tc kernels `fn` launches, from a torch.profiler session.  A session can miss a launch (the first one especially), so `fn` runs
    once before it and three times inside it: the check needs at least one record, and every record must be the expected kernel."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        time.sleep(0.2)  # kernels launched right as a session starts have been seen missing from its trace: start the work 0.2 s in
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "conv_tc" in e.name]


def out_of_scope_case():
    """a 128-channel 3x3 conv with a residual: (inputs, fp64 reference, launcher)"""
    x, w, sc, bi = make(2, 24, 24, 128, 128, 5)
    r = torch.randn(2, 24, 24, 128, generator=torch.Generator().manual_seed(6))
    xp, rp = ops.to_pair(x.to(DEV)), ops.to_pair(r.to(DEV))
    run = lambda: ops.conv2d_pair(xp, _split3_weights(w).to(DEV), sc.to(DEV), bi.to(DEV), pad=1, act=ops.ACT_RELU, residual=rp)
    return ref64(x, w, sc, bi, rp.float().cpu()), run


def dispatch_names():
    """conv_tc kernels launched by an in-scope conv and by the out-of-scope one"""
    x, w, sc, bi = make(2, 24, 24, 32, 64, 3)
    xp = ops.to_pair(x.to(DEV))
    return kernels_run(lambda: conv(xp, w, sc, bi, True)), kernels_run(out_of_scope_case()[1])


def test_dispatch_boundary():
    """Cin = 32 3x3 convs take the small-channel kernel; a 128-channel 3x3 with a residual still runs on the general kernel and is right.  The kernel names
    come from a fresh interpreter: in a process where earlier tests ran profiler sessions, a later session has been seen to record no kernels at all."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import json; from tests.test_gpu_conv_tc_smallc import dispatch_names; print(json.dumps(dispatch_names()))"],
                       cwd=root, capture_output=True, text=True, timeout=150)
    assert r.returncode == 0, r.stderr[-2000:]
    small, general = json.loads(r.stdout.strip().splitlines()[-1])
    assert small and all("conv_tc_smallc_kernel" in n for n in small), small
    assert general and all("conv_tc_kernel" in n and "smallc" not in n for n in general), general
    ref, run = out_of_scope_case()
    check(run().float(), ref)
