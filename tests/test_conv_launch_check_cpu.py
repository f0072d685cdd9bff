"""The per-launch fp64 checker (tests/conv_launch_check.py) proven on a machine without a GPU: around the CPU reference backend every launch of one model
of each family passes in the fp32, fp32_tc and fp16 flows, and each of eight planted kernel errors fails the check at the launch it was planted in."""
import pytest
import torch

from focoos_b200 import ops
from focoos_b200.ops import Pair
from oracle.ops_ref import RefBackend
from tests.conv_launch_check import CheckingBackend, LaunchCheckError, _extent, _flat, seeded_model, synth_batch

# one model of each family, on a small image (odd sizes for the segmenters; DETR needs 300 anchors)
SIZES = {"fai-detr-m-coco": (160, 160), "fai-mf-s-coco-ins": (71, 97), "bisenetformer-s-ade": (71, 97)}


@pytest.fixture()
def backend_reset():
    yield
    ops._backend = None


def _run(name, precision, inner):
    chk = CheckingBackend(inner, f"{name} {precision}")
    ops._backend = chk
    m = seeded_model(name, precision)
    with torch.no_grad():
        m(synth_batch(3, 1, *SIZES[name]))
    return chk


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16"])
@pytest.mark.parametrize("name", list(SIZES))
def test_reference_backend_passes_every_launch(backend_reset, name, precision):
    chk = _run(name, precision, RefBackend())
    assert chk.index > 100 and len(chk.rows) == chk.index
    chk.raise_failures()


# ---- planted errors ---------------------------------------------------------------------------------------------------------------------------------
class Plant:
    """wraps the reference backend and plants one error in the first `op` launch that `when(*args)` accepts: `mutate(fn, *args)` runs in its place"""

    def __init__(self, inner, op, when, mutate):
        self.inner, self.op, self.when, self.mutate = inner, op, when, mutate
        self.checker, self.hit = None, None

    def __getattr__(self, name):
        fn = getattr(self.inner, name)
        if name != self.op:
            return fn

        def call(*a):
            if self.hit is not None or not self.when(*a):
                return fn(*a)
            self.hit = self.checker.index - 1  # the checker numbers the launch before it calls through
            return self.mutate(fn, *a)
        return call


def _drop_tap(fn, x, w, *rest):
    w = w.clone()
    w[:, 0, 2, :] = 0
    return fn(x, w, *rest)


def _ignore_lo(fn, x, *rest):
    buf = x.buf.clone()
    buf[..., x.Ctot + x.c0:x.Ctot + x.c0 + x.C] = 0
    return fn(Pair(buf, x.c0, x.C), *rest)


def _omit_hi_wlo(fn, x, w3, *rest):
    w3 = w3.clone()
    w3[..., x.C:2 * x.C] = 0
    return fn(x, w3, *rest)


def _zero_last_row(fn, *a):
    fn(*a)
    a[8][-1, -1, -1, :] = 0


def _stale_channels(fn, *a):
    out = a[8]
    out[..., -4:] = -1.0  # what the buffer held before the launch (fixed, so that it cannot equal the result by chance)
    stale = out[..., -4:].clone()
    fn(*a)
    out[..., -4:] = stale


def _past_the_view(out):
    """storage offset one pixel pitch past the last element of the output view, if it lies inside the storage"""
    v = out.hi if isinstance(out, Pair) else out
    off = _extent(v)[1] + v.stride(-2)
    return off if off < _flat(v).numel() else None


def _write_past(fn, *a):
    fn(*a)
    out = a[8]
    _flat(out)[_past_the_view(out)] = 777.0


def _residual_after(fn, *a):
    a = list(a)
    a[6] |= 16
    return fn(*a)


def _zero_lo(fn, *a):
    fn(*a)
    a[8].lo.zero_()


def _ragged(x, w, *rest):
    out = rest[6]
    return out.shape[0] * out.shape[1] * out.shape[2] % 128 != 0


# case -> (model, precision, op, when(*args), mutate(fn, *args))
PLANTS = {
    "3x3 tap dropped": ("fai-mf-s-coco-ins", "fp32", "conv2d", lambda x, w, *r: w.dim() == 4 and w.shape[1] == 3, _drop_tap),
    "lo plane of the operand ignored": ("fai-mf-s-coco-ins", "fp32_tc", "conv2d_pair", lambda *a: True, _ignore_lo),
    "hi x W_lo product omitted": ("bisenetformer-s-ade", "fp32_tc", "conv2d_pair", lambda *a: True, _omit_hi_wlo),
    "last row of a ragged tile zeroed": ("bisenetformer-s-ade", "fp16", "conv2d", _ragged, _zero_last_row),
    "last four output channels stale": ("fai-detr-m-coco", "fp32", "conv2d", lambda x, w, *r: w.shape[-4] >= 8, _stale_channels),
    "one value written a pitch past the view": ("fai-detr-m-coco", "fp32", "conv2d", lambda *a: _past_the_view(a[8]) is not None, _write_past),
    "residual after the activation instead of before": ("fai-mf-s-coco-ins", "fp32", "conv2d", lambda *a: a[7] is not None and a[6] == ops.ACT_RELU,
                                                        _residual_after),
    "pair output with a zero lo plane": ("fai-mf-s-coco-ins", "fp32_tc", "conv2d_pair", lambda *a: isinstance(a[8], Pair), _zero_lo),
}


@pytest.mark.parametrize("case", list(PLANTS))
def test_planted_error_fails_at_its_launch(backend_reset, case):
    name, precision, op, when, mutate = PLANTS[case]
    plant = Plant(RefBackend(), op, when, mutate)
    chk = CheckingBackend(plant, f"{name} {precision}")
    plant.checker = chk
    ops._backend = chk
    m = seeded_model(name, precision)
    with torch.no_grad():
        m(synth_batch(3, 1, *SIZES[name]))
    assert plant.hit is not None, f"{case}: no launch to plant it in"
    assert chk.failures, f"{case}: planted at launch #{plant.hit}, the check passed"
    at = f"{name} {precision} launch #{plant.hit} "
    assert all(f.startswith(at) for f in chk.failures), chk.failures[:4]
    with pytest.raises(LaunchCheckError, match=f"launch #{plant.hit} "):
        chk.raise_failures()
