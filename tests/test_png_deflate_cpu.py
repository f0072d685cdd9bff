"""The PNG format the device encoder reproduces, restated on the CPU (oracle/png_ref.py): byte for byte the OpenCV files of tests/golden/png_deflate.npz
(oracle/gen_golden_png_deflate.py), the reference strings of tests/golden/png_masks.json, and cv2.imencode itself on a seeded sweep; and ops.mask_png refusing
host tensors (no CPU fallback)."""
import base64
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import ops
from oracle.gen_golden_png_deflate import load
from oracle.png_ref import mask_png

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _batch(crops, rng, pad=3):
    """crops placed at random offsets in one [n, H, W] uint8 batch of random pixels, with their xyxy boxes (exclusive ends)"""
    H, W = max(c.shape[0] for c in crops) + pad, max(c.shape[1] for c in crops) + pad
    masks = (rng.random((len(crops), H, W)) > 0.5).astype(np.uint8)
    boxes = np.zeros((len(crops), 4), np.int32)
    for i, c in enumerate(crops):
        y, x = int(rng.integers(0, H - c.shape[0] + 1)), int(rng.integers(0, W - c.shape[1] + 1))
        masks[i, y:y + c.shape[0], x:x + c.shape[1]] = c
        boxes[i] = (x, y, x + c.shape[1], y + c.shape[0])
    return torch.from_numpy(masks), torch.from_numpy(boxes)


def _files(data, lengths):
    offs = np.concatenate([[0], np.cumsum(lengths.numpy())])
    return [data[offs[i]:offs[i + 1]] for i in range(len(lengths))]


def test_fixture_covers_the_format():
    g = np.load(os.path.join(GOLDEN, "png_deflate.npz"))
    kinds = [k for t in g["block_types"] for k in str(t).split(",")]
    assert "1" in kinds and "2" in kinds and "0" not in kinds
    assert max(len(str(t).split(",")) for t in g["block_types"]) >= 4
    shapes = [tuple(s) for s in g["shapes"]]
    assert (1, 1) in shapes and (1080, 1920) in shapes and any(w == 1 for _, w in shapes) and any(h == 1 for h, _ in shapes)
    assert "0 stored blocks" in str(g["stored_search"])


def test_reference_reproduces_the_opencv_fixture():
    cases = load()
    masks, boxes = _batch([m.astype(np.uint8) for _, m, _ in cases], np.random.default_rng(0))
    data, lengths = mask_png(masks, boxes)
    for (name, _, png), got in zip(cases, _files(data.numpy().tobytes(), lengths)):
        assert got == png, name


def test_reference_reproduces_the_reference_strings():
    with open(os.path.join(GOLDEN, "png_masks.json")) as f:
        g = json.load(f)
    for k, v in g.items():
        if k == "_meta":
            continue
        m = np.unpackbits(np.array(v["bits"], dtype=np.uint8))[:int(np.prod(v["shape"]))].reshape(v["shape"]).astype(np.uint8)
        data, lengths = mask_png(torch.from_numpy(m)[None], torch.tensor([[0, 0, m.shape[1], m.shape[0]]], dtype=torch.int32))
        assert base64.b64encode(data.numpy().tobytes()).decode() == v["b64"], k


def test_reference_equals_opencv_on_a_seeded_sweep():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    crops = []
    for k in range(120):
        h, w = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        kind = k % 4
        if kind == 0:
            c = rng.random((h, w)) > rng.random()
        elif kind == 1:
            yy, xx = np.mgrid[:h, :w]
            c = np.hypot(yy - h * rng.random(), xx - w * rng.random()) < rng.random() * max(h, w)
        elif kind == 2:
            c = np.tile(np.arange(w) % 2 == 0, (h, 1))
        else:
            c = np.full((h, w), k % 8 == 3)
        crops.append(c.astype(np.uint8))
    masks, boxes = _batch(crops, rng)
    data, lengths = mask_png(masks, boxes)
    for c, got in zip(crops, _files(data.numpy().tobytes(), lengths)):
        assert got == cv2.imencode(".png", c * 255)[1].tobytes(), c.shape


def test_device_encoder_refuses_host_tensors():
    with pytest.raises(RuntimeError):
        ops.mask_png(torch.zeros((1, 4, 4), dtype=torch.uint8), torch.tensor([[0, 0, 4, 4]], dtype=torch.int32))
