"""The per-launch fp64 checker of the fine-tune step (tests/conv_launch_check.py: weight gradients, dilate2, colsum, add_act, and the forward and
data-gradient convs) proven on a machine without a GPU: around the CPU reference backend every launch of one fai-detr-l-coco training step passes in the
fp32, fp32_tc and amp arithmetics, and each of nine planted kernel errors fails the check at the launch it was planted in.

Size: two images of 128x128, whose three memory levels (16x16, 8x8, 4x4) give 336 anchors - at least the 300 queries."""
import pytest
import torch

from focoos_b200 import ops
from oracle.ops_ref import RefBackend
from tests.conv_launch_check import CheckingBackend, LaunchCheckError, train_model, train_step
from tests.test_conv_launch_check_cpu import Plant

B, H, W = 2, 128, 128


@pytest.fixture()
def backend_reset():
    yield
    ops._backend = None


def _step(mode, inner):
    chk = CheckingBackend(inner, f"train {mode}", mode)
    ops._backend = chk
    losses = train_step(train_model(mode), B, H, W)
    assert all(bool(torch.isfinite(v).all()) for v in losses.values())
    return chk


@pytest.mark.parametrize("mode", ["fp32", "fp32_tc", "amp"])
def test_reference_backend_passes_every_launch(backend_reset, mode):
    chk = _step(mode, RefBackend())
    ops_seen = {r["op"] for r in chk.rows}
    assert {"conv2d", "conv_wgrad", "dilate2", "colsum", "add_act"} <= ops_seen, ops_seen
    assert ("conv_wgrad_tc_f16" if mode == "amp" else "conv_wgrad_tc") in ops_seen or mode == "fp32", ops_seen
    assert len(chk.rows) == chk.index > 500
    chk.raise_failures()


# ---- planted errors ---------------------------------------------------------------------------------------------------------------------------------
def _drop_last_image(fn, x, dy, *rest):
    dy = dy.clone()
    dy[-1] = 0
    return fn(x, dy, *rest)


def _drop_dy_lo(fn, x, dy, *rest):
    dy = dy.clone()
    dy[..., dy.shape[-1] // 2:] = 0
    return fn(x, dy, *rest)


def _odd_pixels(fn, x, *rest):
    return fn(torch.roll(x, shifts=(1, 1), dims=(1, 2)), *rest)


def _accumulate(fn, *a):
    prev = a[-1].clone()  # what dw held before the launch
    fn(*a)
    a[-1].add_(prev)


def _round_fp16(fn, *a):
    fn(*a)
    a[-1].copy_(a[-1].half().float())


def _flip_taps(fn, *a):
    fn(*a)
    a[-1].copy_(a[-1].flip(1, 2))


def _junk_last_row(fn, dy, out):
    fn(dy, out)
    out[:, -1] = 1.0


def _miss_last_row(fn, x2d, out):
    return fn(x2d[:-1], out)


def _relu_passes(fn, a, b, dy, act, out):
    fn(a, b, dy, act, out)
    out.copy_(dy)


# case -> (training arithmetic, op, when(*args), mutate(fn, *args))
PLANTS = {
    "weight gradient drops the last image": ("fp32", "conv_wgrad", lambda x, dy, *r: x.shape[0] > 1, _drop_last_image),
    "weight gradient omits hi x dy_lo": ("fp32_tc", "conv_wgrad_tc", lambda *a: True, _drop_dy_lo),
    "stride-2 weight gradient reads the odd pixels": ("fp32_tc", "conv_wgrad_tc", lambda x, dy, KH, KW, s, *r: s == 2, _odd_pixels),
    "weight gradient accumulates into dw": ("fp32_tc", "conv_wgrad_tc", lambda *a: True, _accumulate),
    "amp weight gradient rounded to fp16": ("amp", "conv_wgrad_tc_f16", lambda *a: True, _round_fp16),
    "stem weight gradient with flipped taps": ("fp32", "conv_wgrad", lambda x, dy, KH, KW, s, *r: x.shape[-1] == 3 and s == 2, _flip_taps),
    "dilate2 leaves junk in the last row": ("fp32", "dilate2", lambda *a: True, _junk_last_row),
    "bias gradient misses the last row": ("fp32", "colsum", lambda x2d, out: x2d.shape[0] > 1, _miss_last_row),
    "ReLU gradient passes where the output is zero": ("fp32", "add_act", lambda a, b, dy, act, out: dy is not None and act == ops.ACT_RELU, _relu_passes),
}


@pytest.mark.parametrize("case", list(PLANTS))
def test_planted_error_fails_at_its_launch(backend_reset, case):
    mode, op, when, mutate = PLANTS[case]
    plant = Plant(RefBackend(), op, when, mutate)
    chk = CheckingBackend(plant, f"train {mode}", mode)
    plant.checker = chk
    ops._backend = chk
    train_step(train_model(mode), B, H, W)
    assert plant.hit is not None, f"{case}: no launch to plant it in"
    assert chk.failures, f"{case}: planted at launch #{plant.hit}, the check passed"
    at = f"train {mode} launch #{plant.hit} "
    assert all(f.startswith(at) for f in chk.failures), chk.failures[:4]
    with pytest.raises(LaunchCheckError, match=f"launch #{plant.hit} "):
        chk.raise_failures()
