"""-m gpu: every conv / linear launch of the eleven registry models, in fp32, fp32_tc and fp16, against fp64 of the operands that launch received
(tests/conv_launch_check.py): the SIMT fp32 kernels, the fp16 tensor-core kernels and the fp32-accurate split products, at the layers the models launch -
STDC convs into concat slices, the DETR memory written through a batch stride, the 365- and 80-class heads, the SIMT sigmoid gates, the depthwise stride-2
convs, the per-image mask products at odd sizes.  A census at the end asserts that those configurations were all reached.

Sizes: DETR at 640x640, the MaskFormers and BisenetFormers at 357x483 (odd maps, ragged tiles), two images each; the largest model of each family at
its registry size, one image.  Each launch is followed by a device synchronise and two fp64 convolutions."""
import time

import pytest
import torch

from focoos_b200 import ops
from focoos_b200.model_manager import _REGISTRY
from tests.conv_launch_check import CheckingBackend, seeded_model, summarize, synth_batch
from tests.parity_utils import update_report

# measured on an H100 80GB HBM3 (700 W): 1 to 3 s per case, 70 s for the file (the fp64 references and the per-launch synchronise dominate)
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

PRECISIONS = ["fp32", "fp32_tc", "fp16"]
# (model, B, H, W): every registry model at the size of its family, then the largest of each family at its registry size
CASES = [(name, 2, 640, 640) if r.get("family", "fai_detr") == "fai_detr" else (name, 2, 357, 483) for name, r in _REGISTRY.items()]
CASES += [("fai-detr-l-obj365", 1, 640, 640), ("fai-mf-l-coco-ins", 1, 1024, 1024), ("bisenetformer-l-ade", 1, 640, 640)]
assert len(_REGISTRY) == 11

# the C-ABI entry points CheckingBackend wraps: each wrapped call makes exactly one of these launches
CONV_SYMBOLS = {"fb200_conv2d", "fb200_conv2d_pair", "fb200_linear_rowmax", "fb200_linear_rowmax_pair", "fb200_stem_conv3x3s2", "fb200_stem_conv3x3s2_u8",
                "fb200_dwconv3x3s2_bn"}

# configurations the suite must reach: name -> predicate over a launch row
CENSUS = {
    "stride-2 conv on an odd map": lambda r: r["op"] in ("conv2d", "conv2d_pair") and r["stride"] == 2 and r["odd_map"],
    "flat 1x1 linear": lambda r: r.get("flat_linear", False),
    "per-image weights": lambda r: r.get("per_image", False),
    "96-channel per-image mask product on an odd map": lambda r: r.get("per_image", False) and r["Cin"] == 96 and r["odd_map"],
    "pair output into a channel slice": lambda r: r["fmt"] == "pair" and r.get("out_slice", False),
    "batch-strided output": lambda r: r.get("batch_strided", False),
    "residual before the activation": lambda r: r.get("res") == "pre",
    "residual after the activation": lambda r: r.get("res") == "post",
    "SiLU": lambda r: r.get("act") == ops.ACT_SILU,
    "fp16 GELU": lambda r: r.get("act") == ops.ACT_GELU and r["arith"] == "fp16",
    "SIMT sigmoid": lambda r: r.get("act") == ops.ACT_SIGMOID,
    "small-channel fused 3x3 (32 channels, fp32_tc)": lambda r: r["op"] == "conv2d_pair" and r["Cin"] == 32 and r["k"] == 3 and r["stride"] == 1,
    "365-class head": lambda r: r["Cout"] == 365,
    "80-class head": lambda r: r["Cout"] == 80,
    "linear_rowmax": lambda r: r["op"] == "linear_rowmax",
    "linear_rowmax_pair": lambda r: r["op"] == "linear_rowmax_pair",
    "stem": lambda r: r["op"] == "stem_conv",
    "depthwise stride-2 conv": lambda r: r["op"] == "dwconv3x3s2",
}
_seen = {}   # census item -> the first launch that reached it
_ran = set()


@pytest.fixture()
def checking(monkeypatch):
    """CheckingBackend around the CUDA backend as ops._backend, and a tally of the conv launches that reach the library by any route"""
    tally = []
    call = ops.CudaBackend._call

    def counted(self, name, *args):
        if name in CONV_SYMBOLS:
            tally.append(name)
        return call(self, name, *args)

    monkeypatch.setattr(ops.CudaBackend, "_call", counted)
    chk = CheckingBackend(ops.CudaBackend())
    ops._backend = chk
    try:
        yield chk, tally
    finally:
        ops._backend = None


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,B,H,W", CASES, ids=[f"{n}-b{b}-{h}x{w}" for n, b, h, w in CASES])
def test_every_conv_launch_matches_fp64(checking, name, B, H, W, precision):
    chk, tally = checking
    label = f"{name} b{B} {H}x{W} {precision}"
    m = seeded_model(name, precision, "cuda")
    x = synth_batch(7, B, H, W, "cuda")
    t0 = time.perf_counter()
    chk.begin(label)
    with torch.no_grad():
        m(x)
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    rows = chk.rows
    worst = {k: dict(elem=v[0], elem_at=v[1], agg=v[2], agg_at=v[3]) for k, v in summarize(rows).items()}
    update_report("conv_launches.json", {label: dict(launches=len(rows), seconds=round(secs, 2), worst=worst, rows=rows)})
    for item, pred in CENSUS.items():
        for r in rows:
            if item not in _seen and pred(r):
                _seen[item] = f"{label} #{r['index']} at {r['site']}"
    _ran.add((name, B, H, W, precision))
    assert len(rows) == len(tally) > 0, f"{label}: {len(tally)} conv launches reached the library, {len(rows)} were checked"
    chk.raise_failures()


def test_census_reached_every_configuration():
    """runs after the model cases: each configuration of CENSUS was launched (and so checked) at least once"""
    if len(_ran) < len(CASES) * len(PRECISIONS):
        pytest.skip("needs every case of test_every_conv_launch_matches_fp64 in the same session")
    update_report("conv_launches.json", {"census": _seen})
    missing = [k for k in CENSUS if k not in _seen]
    assert not missing, f"not reached: {missing}"
