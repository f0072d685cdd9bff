"""-m gpu: fai-mf-m-coco-ins and fai-mf-s-coco-ins (128-wide TransformerFPN, 3 encoder layers of 8 heads x 16 channels, 6 masked decoder layers of hidden
256, 128-wide mask features) end to end on the CUDA kernels: against the golden fixtures produced by the unmodified reference (oracle/gen_golden_mf_128.py)
at the bars of tests/test_gpu_mf.py::test_mf_end_to_end_vs_reference_golden, batch invariance at bs=16 800x800, images whose encoder sequence passes the
resident head-dim-16 attention kernels against the CPU oracle, and the public paths (FocoosModel graph replay, TorchScript export)."""
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import ModelManager
from focoos_b200.fai_mf import MaskFormerModelOutput
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import synth_images
from tests.parity_utils import GOLDEN, load_golden, manifest_template, update_report

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]
MODELS = {"fai-mf-m-coco-ins": ("fai_mf_m_coco_ins", 101), "fai-mf-s-coco-ins": ("fai_mf_s_coco_ins", 50)}


def _report(key, val):
    update_report("parity_report_mf_128.json", {key: val})


def _sd(name):
    return seeded_state_dict(manifest_template(MODELS[name][0]), 0)


def _model(name, precision, sd=None):
    m = ModelManager.get(name, state_dict=_sd(name) if sd is None else sd, precision=precision).model
    return m.cuda()


def _batch(imgs):
    return torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs]).cuda()


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16"])
@pytest.mark.parametrize("fixture", ["mf_m_coco_ins_b2_320x416", "mf_s_coco_ins_b2_320x416", "mf_s_coco_ins_b2_357x483"])
def test_mf_128_end_to_end_vs_reference_golden(fixture, precision):
    with open(os.path.join(GOLDEN, "golden_meta_mf_128.json")) as f:
        meta = json.load(f)[fixture]
    g = load_golden(fixture)
    m = _model(meta["model"], precision)
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    taps = {}
    out = m(_batch(imgs), taps=taps)
    torch.cuda.synchronize()
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2).float().cpu()
    ref_pm, pm = g["pred_masks_q10_s2"], pm[:, ::10, ::2, ::2]
    e_logit = float(np.abs(pm.numpy() - ref_pm).max())
    e_cls = float(np.abs(out.logits.cpu().numpy() - g["logits"]).max())
    e_mask = float(np.abs(out.masks[:, ::10, ::4, ::4].cpu().numpy() - g["masks_q10_s4"]).max())
    dets = MaskFormerProcessor(m.config).postprocess(out, imgs, threshold=float(g["threshold"]))
    box_dev = 0
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        if len(d) == n and n:
            box_dev = max(box_dev, int(np.abs(np.array([x.bbox for x in d.detections]) - g["det_boxes"][i, :n]).max()))
    _report(f"{fixture}_{precision}", {"mask_logits_max_abs": e_logit, "mask_logit_scale": scale, "class_prob_max_abs": e_cls, "mask_prob_max_abs": e_mask,
                                       "bbox_max_dev_px": box_dev, "det_count": [len(d) for d in dets], "ref_det_count": g["det_count"].tolist()})
    if precision == "fp16":
        assert np.isfinite(e_logit) and np.isfinite(e_cls) and np.isfinite(e_mask)
        return
    # the bars of the fai-mf-l-coco-ins golden test: fp32 1e-4 * logit scale / 1e-3 / 1e-3; fp32_tc 1e-3 * logit scale / 2e-3 / 2e-3.
    # One exception, stated in DESIGN.md §2: fai-mf-m-coco-ins fp32_tc class probabilities are held to 4e-3.  With the seeded weights its decoder is as
    # peaky as fai-mf-l's (mask logits up to |75|, against |20| for fai-mf-s), and the discrete attention masks (logit < 0) flip on ~1e-5 differences;
    # the measured class-probability deviation is 2.8e-3 on this fixture (H100, 700 W) while the sampled mask logits stay within 1e-4 of their scale, the mask
    # probabilities at 1e-3 and the detections (counts, classes, scores, boxes) equal the reference's.
    cls_bar = 4e-3 if precision == "fp32_tc" and fixture.startswith("mf_m") else 2e-3
    if precision == "fp32":
        assert e_logit <= 1e-4 * scale and e_cls <= 1e-3 and e_mask <= 1e-3, (e_logit, e_cls, e_mask)
    else:
        assert e_logit <= 1e-3 * scale and e_cls <= cls_bar and e_mask <= 2e-3, (e_logit, e_cls, e_mask)
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        if n:
            assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() < 1e-3
    assert box_dev <= 3, box_dev


@pytest.mark.parametrize("name", list(MODELS))
def test_mf_128_bs16_800_batch_invariance(name):
    """bs=16 at 800x800 (625 encoder tokens per image) in fp32_tc: each image's outputs do not depend on the batch they were computed in, bit for bit"""
    m = _model(name, "fp32_tc")
    x = _batch(synth_images(31, [(800, 800)] * 16))
    out16 = m(x)
    out2 = m(x[6:8].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(out16.logits[6:8], out2.logits), "class probabilities depend on the batch"
    assert torch.equal(out16.masks[6:8], out2.masks), "mask probabilities depend on the batch"


@pytest.mark.parametrize("name,size", [("fai-mf-s-coco-ins", (1024, 1024)), ("fai-mf-m-coco-ins", (1024, 1024)), ("fai-mf-s-coco-ins", (1080, 1920))],
                         ids=["s-1024x1024", "m-1024x1024", "s-1080x1920"])
def test_mf_128_large_images_vs_oracle(name, size):
    """The registry's 1024x1024 (1024 encoder tokens) and 1080x1920 (34 x 60 = 2040 tokens: past the resident CUDA-core (1164) and split (1088) head-dim-16
    kernels, which hand over to their streaming kernels) against the CPU oracle, with the bars of test_gpu_mf.py's 1024x1024 test: fp32 encoder memory within
    1e-5 of the oracle's scale, class probabilities 1e-3, mask probabilities 2e-3; fp32_tc encoder memory within 5e-5 (its class / mask probabilities are
    reported: the discrete attention masks of the masked decoder, logit < 0, can flip on 1e-5 differences); detections equal in both.  fp16 runs, finite."""
    from oracle import mf_oracle as O

    sd = _sd(name)
    imgs = synth_images(41, [size])
    x = _batch(imgs)
    cfg = O.MFOracleConfig(depth=MODELS[name][1], feat_dim=128, enc_layers=3, dec_layers=6)
    taps_o = {}
    with torch.no_grad():
        probs, masks = O.mf_forward(sd, x.cpu(), cfg, taps_o)
    proc = ref = None
    for precision in ("fp32", "fp32_tc", "fp16"):
        m = _model(name, precision, sd)
        taps = {}
        out = m(x, taps=taps)
        torch.cuda.synchronize()
        e_cls = float((out.logits.cpu() - probs).abs().max())
        e_mask = float((out.masks.cpu() - masks).abs().max())
        mem = taps["enc_memory"].permute(0, 3, 1, 2).float().cpu()
        e_mem = float((mem - taps_o["enc_memory"]).abs().max() / taps_o["enc_memory"].abs().max())
        _report(f"{name}_{size[0]}x{size[1]}_{precision}", {"enc_memory_rel": e_mem, "class_prob_max_abs": e_cls, "mask_prob_max_abs": e_mask})
        if precision == "fp16":
            assert np.isfinite(e_mem) and np.isfinite(e_cls) and np.isfinite(e_mask)
            continue
        if precision == "fp32":
            assert e_mem <= 1e-5 and e_cls <= 1e-3 and e_mask <= 2e-3, (precision, e_mem, e_cls, e_mask)
        else:
            assert e_mem <= 5e-5, (precision, e_mem)
        proc = proc or MaskFormerProcessor(m.config)
        ref = ref or proc.postprocess(MaskFormerModelOutput(masks=masks.cuda(), logits=probs.cuda(), loss=None), imgs, threshold=0.5)[0]
        got = proc.postprocess(out, imgs, threshold=0.5)[0]
        assert [d.cls_id for d in got.detections] == [d.cls_id for d in ref.detections], precision
        if len(ref.detections):
            assert np.abs(np.array([d.conf for d in got.detections]) - np.array([d.conf for d in ref.detections])).max() < 1e-3
            assert np.abs(np.array([d.bbox for d in got.detections]) - np.array([d.bbox for d in ref.detections])).max() <= 3


@pytest.mark.parametrize("name", list(MODELS))
def test_mf_128_focoos_model_graph_replay_equals_eager(name):
    """ModelManager.get(..., precision="fp32_tc") -> FocoosModel.__call__ on a uint8 batch: the first call runs eagerly, the following ones replay the captured
    CUDA graph - identical detections every time, equal to model.forward + processor.postprocess"""
    fm = ModelManager.get(name, state_dict=_sd(name), precision="fp32_tc")
    fm.model.cuda()
    imgs = synth_images(9, [(320, 416)] * 2)
    runs = [fm(imgs, threshold=0.5, batched=True) for _ in range(3)]
    ref = fm.processor.postprocess(fm.model(_batch(imgs)), imgs, threshold=0.5)
    key = lambda dets: [[(d.cls_id, tuple(d.bbox), d.mask) for d in r.detections] for r in dets]  # noqa: E731
    assert key(runs[0]) == key(runs[1]) == key(runs[2]) == key(ref)
    for a, b in zip(runs[2], ref):
        assert np.allclose([d.conf for d in a.detections], [d.conf for d in b.detections], atol=1e-6)


@pytest.mark.parametrize("name", list(MODELS))
def test_mf_128_torchscript_roundtrip_equals_eager(name, tmp_path):
    """FocoosModel.export -> torch.jit.load: the file's meta (asdict(config)) rebuilds the 128-wide model; same tensors as the eager model, and the exported
    model serves the same detections through the processor"""
    fm = ModelManager.get(name, state_dict=_sd(name), precision="fp32_tc")
    fm.model.cuda()
    im = fm.export(out_dir=str(tmp_path), image_size=320)
    imgs = synth_images(13, [(320, 416)] * 2)
    x = _batch(imgs)
    eager = fm.model(x)
    masks, logits = torch.jit.load(str(tmp_path / "model.pt"))(x)
    assert torch.equal(masks, eager.masks) and torch.equal(logits, eager.logits)
    # the exported graph returns the materialised masks, FocoosModel the low-resolution logits its post-process upsamples itself: same detections,
    # scores to fp32 reassociation
    d1, d2 = im.infer(imgs[0], threshold=0.5), fm.infer(imgs[0], threshold=0.5)
    assert [(d.cls_id, d.bbox, d.mask) for d in d1.detections] == [(d.cls_id, d.bbox, d.mask) for d in d2.detections]
    assert np.allclose([d.conf for d in d1.detections], [d.conf for d in d2.detections], rtol=1e-5)


def test_mf_s_infer_returns_detections():
    """the public one-liner on the registry entry: ModelManager.get("fai-mf-s-coco-ins") (default precision) -> infer(image) -> detections with masks"""
    fm = ModelManager.get("fai-mf-s-coco-ins", state_dict=_sd("fai-mf-s-coco-ins"))
    fm.model.cuda()
    img = synth_images(3, [(480, 640)])[0]
    dets = fm.infer(img, threshold=0.3)
    assert len(dets.detections) > 0
    for d in dets.detections:
        assert 0 <= d.cls_id < 80 and 0.3 <= d.conf <= 1 and d.mask is not None
