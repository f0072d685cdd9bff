"""-m gpu: the device PNG encoder (fb200_mask_png) against the OpenCV files of tests/golden/png_deflate.npz, all masks in one call and one at a time; against
the CPU restatement (oracle/png_ref.py) on a seeded batch of mixed crops; and, through FocoosModel.__call__ (graph replay) and MaskFormerProcessor.postprocess on the lazy and
the materialised mask paths, the same detections (class, box, confidence, mask string) as the host tail it replaces applied to the same device masks."""
import base64

import numpy as np
import pytest
import torch

from focoos_b200 import ModelManager, ops
from focoos_b200.processor import binary_mask_to_base64
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import synth_images
from oracle.gen_golden_png_deflate import load
from oracle.png_ref import mask_png
from tests.parity_utils import manifest_template
from tests.test_png_deflate_cpu import _batch, _files

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _encode(masks, boxes):
    data, lengths = ops.mask_png(masks.cuda(), boxes.cuda())
    return _files(data.cpu().numpy().tobytes(), lengths)


def test_fixture_in_one_call_and_one_at_a_time():
    cases = load()
    masks, boxes = _batch([m.astype(np.uint8) for _, m, _ in cases], np.random.default_rng(0))
    for (name, _, png), got in zip(cases, _encode(masks, boxes)):
        assert got == png, name
    for name, m, png in cases:
        (got,) = _encode(torch.from_numpy(m.astype(np.uint8))[None], torch.tensor([[0, 0, m.shape[1], m.shape[0]]], dtype=torch.int32))
        assert got == png, name


def test_matches_the_cpu_reference_on_mixed_crops():
    rng = np.random.default_rng(9)
    n, H, W = 200, 120, 160
    yy, xx = np.mgrid[:H, :W]
    masks = np.zeros((n, H, W), np.uint8)
    for i in range(n):
        kind = i % 5
        if kind == 0:
            masks[i] = rng.random((H, W)) > rng.random()
        elif kind == 1:
            masks[i] = np.hypot(yy - H * rng.random(), xx - W * rng.random()) < rng.random() * 90
        elif kind == 2:
            masks[i] = (xx + i) % 2
        elif kind == 3:
            masks[i] = i % 2
        else:
            masks[i] = (rng.random((H, 1)) > 0.5) & (rng.random((1, W)) > 0.3)
    x1, y1 = rng.integers(0, W, n), rng.integers(0, H, n)
    boxes = np.stack([x1, y1, x1 + rng.integers(0, W + 5, n), y1 + rng.integers(0, H + 5, n)], 1).astype(np.int32)
    boxes[::17, 2] = boxes[::17, 0]  # crops without columns
    boxes[::13, 2] = boxes[::13, 0] + 1  # one pixel wide
    masks_t, boxes_t = torch.from_numpy(masks), torch.from_numpy(boxes)
    want, want_len = mask_png(masks_t, boxes_t)
    data, lengths = ops.mask_png(masks_t.cuda(), boxes_t.cuda())
    assert torch.equal(lengths, want_len)
    assert data.cpu().numpy().tobytes() == want.numpy().tobytes()


MANIFESTS = {"fai-mf-l-coco-ins": "fai_mf_l_coco_ins", "fai-mf-s-coco-ins": "fai_mf_s_coco_ins", "fai-mf-m-ade": "fai_mf_m_ade",
             "bisenetformer-s-ade": "bisenetformer_s_ade"}


def _host_tail_mask_png(masks, boxes):
    """the tail this encoder replaces, as a drop-in for ops.mask_png: the masks copied to the host, cropped and encoded there one at a time"""
    m, box = masks.cpu().numpy().astype(bool), boxes.cpu().numpy()
    files = []
    for i in range(len(m)):
        x1, y1, x2, y2 = (int(v) for v in box[i])
        crop = m[i][y1:min(y2, m[i].shape[0]), x1:min(x2, m[i].shape[1])]
        files.append(base64.b64decode(binary_mask_to_base64(crop)) if crop.size else b"")
    lengths = torch.tensor([len(f) for f in files], dtype=torch.int32)
    return torch.frombuffer(bytearray(b"".join(files) or b"\0"), dtype=torch.uint8)[:int(lengths.sum())], lengths


def _run(fn):
    """detections, or the name of the exception: a kept mask whose crop has no rows or no columns makes cv2.imencode raise, with the old tail as with this one"""
    try:
        return fn()
    except Exception as e:  # noqa: BLE001
        return type(e).__name__


def _same(a, b):
    """class, box and mask string identical; confidence to 1e-6 (the mask-score reduction sums with atomics, so two post-processes differ in the last bits)"""
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    key = lambda dets: [[(d.cls_id, tuple(d.bbox), d.mask) for d in r.detections] for r in dets]  # noqa: E731
    return key(a) == key(b) and all(np.allclose([d.conf for d in x.detections], [d.conf for d in y.detections], rtol=0, atol=1e-6) for x, y in zip(a, b))


@pytest.mark.parametrize("precision", ["fp32_tc", "fp16"])
@pytest.mark.parametrize("name", list(MANIFESTS))
def test_model_detections_equal_the_host_tail(name, precision, monkeypatch):
    pytest.importorskip("cv2")
    fm = ModelManager.get(name, state_dict=seeded_state_dict(manifest_template(MANIFESTS[name]), 0), precision=precision)
    fm.model.cuda()
    kept = 0
    for size in [(320, 416), (1080, 1920)]:
        imgs = synth_images(21, [size] * 2)
        runs = [_run(lambda: fm(imgs, threshold=0.3, batched=True)) for _ in range(2)]  # eager, then CUDA-graph replay
        assert _same(runs[0], runs[1]), size
        x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs]).cuda()
        for lazy in (True, False):
            fm.model.lazy_masks = lazy
            out = fm.model(x)
            new = _run(lambda: fm.processor.postprocess(out, imgs, threshold=0.3))
            with monkeypatch.context() as mp:
                mp.setattr(ops, "mask_png", _host_tail_mask_png)
                old = _run(lambda: fm.processor.postprocess(out, imgs, threshold=0.3))
            assert _same(new, old), (size, lazy)
            if lazy:
                assert _same(new, runs[1]), size
            kept += 0 if isinstance(new, str) else sum(len(r.detections) for r in new)
        fm.model.lazy_masks = False
    assert kept > 0
