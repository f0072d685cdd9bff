"""-m gpu: the ADE20K semantic segmenters (fai-mf-l-ade, fai-mf-m-ade, bisenetformer-m-ade, bisenetformer-s-ade) on the CUDA kernels: the two tensor-core
configurations bisenetformer-m-ade is the first to run (the per-image mask product on 96 channels, the 256 -> 96 mask-MLP output linear) against fp64, the
models end to end against the golden fixtures produced by the unmodified reference (oracle/gen_golden_ade.py), batch invariance at bs=16 640x640, and the
public paths (FocoosModel graph replay, TorchScript export, ModelManager.get(name).infer)."""
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import ModelManager, ops
from focoos_b200.engine import _split3_weights
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import synth_images
from tests.parity_utils import GOLDEN, load_golden, manifest_template, update_report

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]
DEV = "cuda"
MANIFESTS = {"fai-mf-l-ade": "fai_mf_l_ade", "fai-mf-m-ade": "fai_mf_m_ade", "bisenetformer-m-ade": "bisenetformer_m_ade",
             "bisenetformer-s-ade": "bisenetformer_s_ade"}
FIXTURES = ["mf_l_ade_b2_320x416", "mf_m_ade_b2_320x416", "mf_m_ade_b2_357x483", "bisenetformer_m_ade_b2_256x384", "bisenetformer_m_ade_b2_357x483",
            "bisenetformer_s_ade_b2_256x384"]


def rnd(shape, dtype, seed, s=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * s).to(dtype)


def close(a, b, tol, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    err, scale = float((a - b).abs().max()), max(1.0, float(b.abs().max()))
    assert err <= tol * scale, f"{what}: max|d|={err:.3e} scale={scale:.2e}"


def _report(key, val):
    update_report("parity_report_ade.json", {key: val})


def _sd(name):
    return seeded_state_dict(manifest_template(MANIFESTS[name]), 0)


def _model(name, precision):
    return ModelManager.get(name, state_dict=_sd(name), precision=precision).model.cuda()


def _batch(imgs):
    return torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs]).cuda()


# ---- the two tensor-core configurations of bisenetformer-m-ade --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,h,w", [(2, 80, 80), (2, 45, 61)], ids=["80x80", "45x61"])
def test_per_image_mask_product_96_channels(B, h, w):
    """einsum("bqc,bchw->bqhw") on 96 mask-feature channels (bisenetformer-m-ade) on the fp32-accurate tensor-core path: fb200_conv2d_pair with a weight batch
    stride and 32-channel chunks (three per plane, the 64-byte swizzle, the 3-D weight map) vs fp64, into the first Q columns of a padded NHWC buffer like
    MFEngine._heads does"""
    C, Q = 96, 100
    x, me = rnd((B, h, w, C), torch.float32, 11), rnd((B, Q, C), torch.float32, 12, 0.5)
    ref = torch.einsum("bqc,bhwc->bhwq", me.double(), x.double())
    Qp = (Q + 7) // 8 * 8
    out = torch.zeros((B, h, w, Qp), dtype=torch.float32, device=DEV)
    ops.conv2d_per_image(ops.to_pair(x.to(DEV)), _split3_weights(me.to(DEV)).reshape(B, Q, 1, 1, 3 * C), out=out[..., :Q])
    close(out[..., :Q], ref, 2e-5, "per-image mask product, C=96 (split)")
    assert float(out[..., Q:].abs().max()) == 0.0, "the padding columns of the buffer must stay untouched"


@pytest.mark.parametrize("out_pair", [False, True], ids=["fp32_out", "pair_out"])
def test_mask_mlp_output_linear_256_to_96(out_pair):
    """the mask-MLP output layer of bisenetformer-m-ade, 256 -> 96 (N = 96 inside a 128-wide tile), on the pair operand vs fp64, with fp32 or pair output"""
    B, Q, K, N = 2, 100, 256, 96
    x, w, b = rnd((B, Q, K), torch.float32, 21), rnd((N, K), torch.float32, 22, 0.06), rnd((N,), torch.float32, 23, 0.1)
    ref = x.double() @ w.double().t() + b.double()
    y = ops.linear_pair(ops.to_pair(x.to(DEV)), _split3_weights(w.to(DEV)), b.to(DEV), out_pair=out_pair)
    assert tuple(y.shape) == (B, Q, N)
    # the pair output holds the fp32 result as fp16 hi + lo, which keeps ~2^-22 of it
    close(y.float(), ref, 2e-5, f"linear 256->96 ({'pair' if out_pair else 'fp32'} output)")


# ---- the models ----------------------------------------------------------------------------------------------------------------------------------------
# Stated exceptions (DESIGN.md §2): the masked decoder turns tiny differences into flipped attention-mask bits (logit < 0), which the seeded, peaky weights
# amplify.
#  * fai-mf-l-ade (mask logits up to |130|) is chaotic on its golden: its fp32 flow on the CPU, fed the same images times (1 + 1e-6 noise), moves the class
#    probabilities by 0.07 and the mask probabilities by 0.23 while its mask features move by 4e-6.  fp32 meets the bars (class probabilities 5.8e-4 off,
#    H100, 700 W); fp32_tc (mask features 1.4e-4 off) lands inside that spread (class 0.070, masks 0.21) and is held to the mask-feature tap and to the spread.
#  * fai-mf-m-ade at 357x483: flipped bits put the class probabilities 2.9e-3 (fp32) and 1.06e-2 (fp32_tc) off, H100, 700 W; held to 4e-3 / 2e-2.  Mask
#    logits, mask probabilities and detections meet the bars.
CHAOTIC = {("mf_l_ade_b2_320x416", "fp32_tc")}
CLS_BAR = {("mf_m_ade_b2_357x483", "fp32"): 4e-3, ("mf_m_ade_b2_357x483", "fp32_tc"): 2e-2}


def _masks_sample(g, masks):
    key = "masks_q10_s4" if "masks_q10_s4" in g else "masks_q20_s4"  # odd-size files hold every 20th query
    return masks[:, ::(10 if key == "masks_q10_s4" else 20), ::4, ::4], g[key]


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16"])
@pytest.mark.parametrize("fixture", FIXTURES)
def test_ade_end_to_end_vs_reference_golden(fixture, precision):
    with open(os.path.join(GOLDEN, "golden_meta_ade.json")) as f:
        meta = json.load(f)[fixture]
    g = load_golden(fixture)
    m = _model(meta["model"], precision)
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    taps = {}
    out = m(_batch(imgs), taps=taps)
    torch.cuda.synchronize()
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2).float().cpu()
    e_logit = float(np.abs(pm[:, ::10, ::2, ::2].numpy() - g["pred_masks_q10_s2"]).max())
    e_cls = float(np.abs(out.logits.cpu().numpy() - g["logits"]).max())
    got, ref = _masks_sample(g, out.masks)
    e_mask = float(np.abs(got.cpu().numpy() - ref).max())
    e_mf = None
    if "mask_features_tap" in g:
        mf = taps["mask_features"].permute(0, 3, 1, 2)[:, ::16, ::4, ::4].float().cpu().numpy()
        e_mf = float(np.abs(mf - g["mask_features_tap"]).max() / np.abs(g["mask_features_tap"]).max())
    dets = MaskFormerProcessor(m.config).postprocess(out, imgs, threshold=float(g["threshold"]))
    _report(f"{fixture}_{precision}", {"mask_logits_max_abs": e_logit, "mask_logit_scale": scale, "class_prob_max_abs": e_cls, "mask_prob_max_abs": e_mask,
                                       "mask_features_rel": e_mf, "det_count": [len(d) for d in dets], "ref_det_count": g["det_count"].tolist()})
    if precision == "fp16":
        assert np.isfinite(e_logit) and np.isfinite(e_cls) and np.isfinite(e_mask)
        return
    fp32 = precision == "fp32"
    if e_mf is not None:
        assert e_mf <= (1e-4 if fp32 else 1e-3), e_mf
    if (fixture, precision) in CHAOTIC:
        assert e_logit <= 0.05 * scale and e_cls <= 0.1 and e_mask <= 0.3, (e_logit, e_cls, e_mask)
        return
    if fixture.startswith("mf_"):  # the bars of test_gpu_mf_128.py
        cls_bar = CLS_BAR.get((fixture, precision), 1e-3 if fp32 else 2e-3)
        if fp32:
            assert e_logit <= 1e-4 * scale and e_cls <= cls_bar and e_mask <= 1e-3, (e_logit, e_cls, e_mask)
        else:
            assert e_logit <= 1e-3 * scale and e_cls <= cls_bar and e_mask <= 2e-3, (e_logit, e_cls, e_mask)
    else:  # the bars of test_gpu_bisenet.py
        assert e_logit <= (1e-4 if fp32 else 2e-4) * scale and e_cls <= 1e-3 and e_mask <= 1e-3, (e_logit, e_cls, e_mask)
    for i, d in enumerate(dets):  # semantic detections: the reference's counts and labels, scores within 1e-3, boxes within 3 px
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        if n:
            assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() < 1e-3
            assert np.abs(np.array([x.bbox for x in d.detections]) - g["det_boxes"][i, :n]).max() <= 3


@pytest.mark.parametrize("name", list(MANIFESTS))
def test_ade_bs16_640_batch_invariance(name):
    """bs=16 at 640x640 in fp32_tc: each image's outputs do not depend on the batch they were computed in, bit for bit"""
    m = _model(name, "fp32_tc")
    x = _batch(synth_images(31, [(640, 640)] * 16))
    out16 = m(x)
    out2 = m(x[6:8].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(out16.logits[6:8], out2.logits), "class probabilities depend on the batch"
    assert torch.equal(out16.masks[6:8], out2.masks), "mask probabilities depend on the batch"


@pytest.mark.parametrize("name", list(MANIFESTS))
def test_ade_focoos_model_graph_replay_equals_eager(name):
    """FocoosModel.__call__ on a uint8 batch (fp32_tc): the first call runs eagerly, the next two replay the captured CUDA graph - identical detections every
    time, equal to model.forward + processor.postprocess"""
    fm = ModelManager.get(name, state_dict=_sd(name), precision="fp32_tc")
    fm.model.cuda()
    imgs = synth_images(9, [(320, 416)] * 2)
    runs = [fm(imgs, threshold=0.5, batched=True) for _ in range(3)]
    ref = fm.processor.postprocess(fm.model(_batch(imgs)), imgs, threshold=0.5)
    key = lambda dets: [[(d.cls_id, tuple(d.bbox), d.mask) for d in r.detections] for r in dets]  # noqa: E731
    assert key(runs[0]) == key(runs[1]) == key(runs[2]) == key(ref)
    for a, b in zip(runs[2], ref):
        assert np.allclose([d.conf for d in a.detections], [d.conf for d in b.detections], atol=1e-6)


@pytest.mark.parametrize("name", ["fai-mf-m-ade", "bisenetformer-m-ade"])
def test_ade_torchscript_roundtrip_equals_eager(name, tmp_path):
    """FocoosModel.export -> torch.jit.load: the file's meta rebuilds the model (fai-mf-m-ade with its STDC trunk); same tensors as the eager model, and the
    exported model serves the same detections through the processor"""
    fm = ModelManager.get(name, state_dict=_sd(name), precision="fp32_tc")
    fm.model.cuda()
    im = fm.export(out_dir=str(tmp_path), image_size=320)
    imgs = synth_images(13, [(320, 416)] * 2)
    x = _batch(imgs)
    eager = fm.model(x)
    masks, logits = torch.jit.load(str(tmp_path / "model.pt"))(x)
    assert torch.equal(masks, eager.masks) and torch.equal(logits, eager.logits)
    d1, d2 = im.infer(imgs[0], threshold=0.5), fm.infer(imgs[0], threshold=0.5)
    assert [(d.cls_id, d.bbox, d.mask) for d in d1.detections] == [(d.cls_id, d.bbox, d.mask) for d in d2.detections]
    assert np.allclose([d.conf for d in d1.detections], [d.conf for d in d2.detections], rtol=1e-5)


@pytest.mark.parametrize("name", list(MANIFESTS))
def test_ade_infer_returns_semantic_detections(name):
    """the public one-liner on the registry entry: ModelManager.get(name) (default precision) -> infer(image) -> semantic detections with masks"""
    fm = ModelManager.get(name, state_dict=_sd(name))
    fm.model.cuda()
    img = synth_images(3, [(480, 640)])[0]
    dets = fm.infer(img, threshold=0.3)
    assert len(dets.detections) > 0
    for d in dets.detections:
        assert 0 <= d.cls_id < 150 and 0.3 <= d.conf <= 1 and d.mask is not None
