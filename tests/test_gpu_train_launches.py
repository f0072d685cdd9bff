"""-m gpu: every conv / linear launch of one fai-detr-l-coco fine-tune step - forward, data gradient, weight gradient - and the dilate2, colsum and
add_act launches of its backward, against fp64 of the operands each launch received (tests/conv_launch_check.py).  The step is the trainer's: seeded
weights with desaturated classifiers, synthetic images and targets, forward, criterion, loss-scaled backward, clipped AdamW.

Cases: bs=16 at 640x640 (the fine-tune shape: 1.6 M pixels per weight element in the stem's 32-channel convs, 134,400 memory rows in the linears) in
amp (the trainer's default arithmetic), fp32_tc and fp32; bs=3 at 544x736 (17x23 and 34x46 maps in the deep stages); bs=1 at 640x640 in fp32_tc, where
the 20x20 maps have fewer than 512 pixels and the weight gradient falls back to the CUDA-core kernel.  A census at the end asserts that the configurations
where these kernels could go wrong were all reached.

Measured on an H100 80GB HBM3 (700 W): 800 checked launches per case; the step with its checks takes 6.8 s (amp), 2.9 s (fp32_tc) and 3.1 s (fp32)
at bs=16, 2.1 s at bs=3 and 1.2 s at bs=1, 30 s for the file.  Each launch is followed by a device synchronise and its fp64 references; the weight
gradient's reference is one fp64 GEMM per filter tap, 2-4x faster there than cuDNN's fp64 backward-filter (5.6 vs 9.9 ms at 16x320x320x32, 3x3)."""
import time

import pytest
import torch

from focoos_b200 import ops
from tests.conv_launch_check import CheckingBackend, summarize, train_model, train_step
from tests.parity_utils import update_report

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

# (training arithmetic, B, H, W)
CASES = [("amp", 16, 640, 640), ("fp32_tc", 16, 640, 640), ("fp32", 16, 640, 640), ("fp32_tc", 3, 544, 736), ("fp32_tc", 1, 640, 640)]

# the C-ABI entry points of the wrapped operators: each wrapped call makes exactly one of these launches
SYMBOLS = {"fb200_conv2d", "fb200_conv2d_pair", "fb200_conv_wgrad", "fb200_conv_wgrad_tc", "fb200_conv_wgrad_tc_f16", "fb200_dilate2", "fb200_colsum",
           "fb200_add_act"}


def _backward(r):
    return ".backward:" in r["site"]


def _tc(r):
    return r["mode"] in ("fp32_tc", "amp")


# configurations the step must reach: name -> predicate over a launch row
CENSUS = {
    "stem weight gradient 3->32 3x3 s2 (dedicated kernel)": lambda r: r["op"] == "conv_wgrad" and r["kernel"] == "stem" and r["Cin"] == 3 and r["Cout"] == 32,
    "split weight gradient k3 s1": lambda r: r["op"] == "conv_wgrad_tc" and r["k"] == 3 and r["stride"] == 1,
    "split weight gradient k1": lambda r: r["op"] == "conv_wgrad_tc" and r["k"] == 1,
    "split weight gradient k3 s2": lambda r: r["op"] == "conv_wgrad_tc" and r["k"] == 3 and r["stride"] == 2,
    "split weight gradient, 32 channels (half a TMA box)": lambda r: r["op"] == "conv_wgrad_tc" and r["Cin"] == 32,
    "f16 weight gradient k3 s1": lambda r: r["op"] == "conv_wgrad_tc_f16" and r["k"] == 3 and r["stride"] == 1,
    "f16 weight gradient k3 s2": lambda r: r["op"] == "conv_wgrad_tc_f16" and r["k"] == 3 and r["stride"] == 2,
    "f16 weight gradient k1": lambda r: r["op"] == "conv_wgrad_tc_f16" and r["k"] == 1,
    "CUDA-core weight gradient in a tensor-core mode: K=4 query_pos_head layer 0": lambda r: r["op"] == "conv_wgrad" and _tc(r) and r["linear"] and r["Cin"] == 4,
    "CUDA-core weight gradient in a tensor-core mode: Cout=4 box head": lambda r: r["op"] == "conv_wgrad" and _tc(r) and r["linear"] and r["Cout"] == 4,
    "CUDA-core weight gradient in a tensor-core mode: B*Ho*Wo < 512": lambda r: (r["op"] == "conv_wgrad" and _tc(r) and r["K"] < 512 and r["Cin"] % 8 == 0
                                                                                and r["Cout"] % 8 == 0),
    "linear weight gradient over >= 100k rows": lambda r: r["op"].startswith("conv_wgrad") and r["linear"] and r["K"] >= 100_000,
    "stride-2 data gradient through dilate2, fp32": lambda r: r["op"] == "dilate2" and r["mode"] == "fp32",
    "stride-2 data gradient through dilate2, fp32_tc": lambda r: r["op"] == "dilate2" and r["mode"] == "fp32_tc",
    "stride-2 data gradient through dilate2, amp": lambda r: r["op"] == "dilate2" and r["mode"] == "amp",
    "pair data-gradient conv": lambda r: r["op"] == "conv2d_pair" and _backward(r),
    "fp16-operand data-gradient conv, fp32 output": lambda r: r["op"] == "conv2d" and r["arith"] == "fp16" and r["fmt"] == "fp32" and _backward(r),
    "bias gradient of the 80-class head": lambda r: r["op"] == "colsum" and r["Cout"] == 80,
    "ReLU gradient gate": lambda r: r["op"] == "add_act" and r["grad"] and r["act"] == ops.ACT_RELU,
    "GELU forward": lambda r: r["op"] == "add_act" and not r["grad"] and r["act"] == ops.ACT_GELU,
    "GELU gradient": lambda r: r["op"] == "add_act" and r["grad"] and r["act"] == ops.ACT_GELU,
}
_seen = {}   # census item -> the first launch that reached it and passed its checks
_ran = set()


@pytest.fixture()
def checking(monkeypatch):
    """CheckingBackend around the CUDA backend as ops._backend, and a tally of the wrapped launches that reach the library by any route"""
    tally = []
    call = ops.CudaBackend._call

    def counted(self, name, *args):
        if name in SYMBOLS:
            tally.append(name)
        return call(self, name, *args)

    monkeypatch.setattr(ops.CudaBackend, "_call", counted)
    chk = CheckingBackend(ops.CudaBackend())
    ops._backend = chk
    try:
        yield chk, tally
    finally:
        ops._backend = None


@pytest.mark.parametrize("mode,B,H,W", CASES, ids=[f"{m}-b{b}-{h}x{w}" for m, b, h, w in CASES])
def test_every_train_step_launch_matches_fp64(checking, mode, B, H, W):
    chk, tally = checking
    label = f"fai-detr-l-coco train b{B} {H}x{W} {mode}"
    m = train_model(mode, "cuda")
    torch.cuda.synchronize()
    tally.clear()
    t0 = time.perf_counter()
    chk.begin(label, mode)
    losses = train_step(m, B, H, W, "cuda")
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    rows = chk.rows
    worst = {k: dict(elem=v[0], elem_at=v[1], agg=v[2], agg_at=v[3]) for k, v in summarize(rows).items()}
    update_report("train_launches.json", {label: dict(launches=len(rows), seconds=round(secs, 2), worst=worst, rows=rows)})
    for item, pred in CENSUS.items():
        for r in rows:
            if item not in _seen and r["ok"] and pred(r):
                _seen[item] = f"{label} #{r['index']} at {r['site']}"
    _ran.add((mode, B, H, W))
    print(f"{label}: {len(rows)} launches in {secs:.1f} s; worst {worst}")
    assert all(bool(torch.isfinite(v).all()) for v in losses.values())
    assert len(rows) == len(tally) > 0, f"{label}: {len(tally)} wrapped launches reached the library, {len(rows)} were checked"
    chk.raise_failures()


def test_census_reached_every_configuration():
    """runs after the step cases: each configuration of CENSUS was launched, and passed its checks, at least once"""
    if len(_ran) < len(CASES):
        pytest.skip("needs every case of test_every_train_step_launch_matches_fp64 in the same session")
    update_report("train_launches.json", {"census": _seen})
    missing = [k for k in CENSUS if k not in _seen]
    assert not missing, f"not reached: {missing}"
