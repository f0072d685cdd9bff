"""Semantic evaluation without a GPU: MaskFormerProcessor.eval_postprocess + SemSegEvaluator on the CPU reference backend against the stored output of the
UNMODIFIED reference's processor and SemSegEvaluator (tests/golden/sem_seg_eval_proc.npz, oracle/gen_golden_sem_seg_eval.py) with the CPU operators of
oracle/sem_seg_ref.py, the CPU operator of the confusion kernel against numpy argmax + bincount, the refusal of instance configs, and the unchanged detection path of inference_on_dataset."""
import os

import numpy as np
import pytest
import torch

from focoos_b200 import ops
from focoos_b200.fai_mf import LazyMasks, MaskFormerConfig, MaskFormerModelOutput
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.trainer import BoxAPEvaluator, SemSegEvaluator, SyntheticDetectionDataset, SyntheticSemSegDataset, inference_on_dataset
from oracle.sem_seg_ref import SemSegRefBackend

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODEL_CASES = ["bisenetformer-s-ade", "fai-mf-m-ade"]


def _gt(g, H, W, C=150):
    """class blocks on a 6x6 grid, ~5% ignore (255) pixels and a few pixels labelled C (counted in the ignore column, as the reference's bincount does)"""
    blocks = torch.randint(0, C, (6, 6), generator=g)
    gt = blocks[(torch.arange(H) * 6 // H)[:, None], (torch.arange(W) * 6 // W)[None, :]]
    r = torch.rand((H, W), generator=g)
    gt[r < 0.05] = 255
    gt[r > 0.995] = C
    return gt.numpy().astype(np.uint8)


def _case(seed=0):
    """(low-resolution mask logits NHWC [3,16,24,104], class probabilities [3,100,150], entries, ground truths): input 64x96, the third entry evaluated at
    50x75; class 7 duplicates class 3 (exact ties: the first maximum wins), class 11 is class 5 scaled by 1 + 2^-16 (near ties)"""
    g = torch.Generator().manual_seed(seed)
    B, Q, C, H, W = 3, 100, 150, 64, 96
    low = torch.randn((B, H // 4, W // 4, 104), generator=g) * 3
    low[..., Q:] = 0
    logits = torch.softmax(torch.randn((B, Q, C + 1), generator=g) * 2, -1)[..., :-1].contiguous()
    logits[:, :, 7] = logits[:, :, 3]
    logits[:, :, 11] = logits[:, :, 5] * (1 + 2 ** -16)
    sizes = [(H, W), (H, W), (50, 75)]
    entries = [{"image_size": (H, W), "height": h, "width": w} for h, w in sizes]
    gts = [_gt(g, h, w) for h, w in sizes]
    return low, logits, entries, gts


def _model_case():
    """(images HWC uint8, entries, ground truths) of the model goldens: two 256x384 images and one 357x483 image"""
    from oracle.gen_golden import synth_images
    sizes = [(256, 384), (256, 384), (357, 483)]
    imgs = synth_images(11, sizes)
    g = torch.Generator().manual_seed(11)
    return imgs, [{"image_size": s, "height": s[0], "width": s[1]} for s in sizes], [_gt(g, *s) for s in sizes]


def golden_metrics(z):
    return {str(k): (None if np.isnan(v) else float(v)) for k, v in zip(z["metric_keys"], z["metric_vals"])}


@pytest.fixture()
def ref_backend():
    ops._backend = SemSegRefBackend()
    yield
    ops._backend = None


def _proc():
    return MaskFormerProcessor(MaskFormerConfig(num_classes=150, postprocessing_type="semantic", predict_all_pixels=True, use_mask_score=False))


def test_processor_and_evaluator_match_the_reference(ref_backend):
    z = np.load(os.path.join(GOLDEN, "sem_seg_eval_proc.npz"))
    low, logits, entries, gts = _case()
    out = _proc().eval_postprocess(MaskFormerModelOutput(masks=LazyMasks(low, 100, (64, 96)), logits=logits), entries)
    assert [tuple(o["sem_seg"].shape) for o in out] == [(150, 64, 96), (150, 64, 96), (150, 50, 75)]
    for i, o in enumerate(out):
        assert np.array_equal(o["sem_seg"].argmax(0).numpy(), z[f"pred_{i}"])
    ev = SemSegEvaluator(150)
    ev.reset()
    ev.process([{"sem_seg": gt} for gt in gts], out)
    assert np.array_equal(ev.confusion_matrix(), z["conf"])
    assert ev.evaluate() == {"sem_seg": golden_metrics(z)}


def test_reference_confusion_operator_matches_bincount_of_argmax():
    g = torch.Generator().manual_seed(1)
    B, H, W, Cp, C = 2, 9, 13, 12, 10
    scores = torch.randint(0, 4, (B, H, W, Cp), generator=g).float()  # many exact ties
    scores[0, 0, 0, 3] = float("nan")
    scores[1, 2, 2, [4, 6]] = float("nan")  # the first NaN wins
    labels = torch.randint(0, C + 1, (B, H, W), generator=g, dtype=torch.int32)
    labels[0, 1] = 255
    labels[1, 3, :4] = -3  # invalid: not counted, reported
    conf = torch.zeros((C + 1, C + 1), dtype=torch.int64)
    inv = torch.zeros((1,), dtype=torch.int64)
    SemSegRefBackend()._sem_seg_confusion(scores, labels, C, 255, conf, inv)
    pred = np.argmax(scores[..., :C].numpy(), -1).reshape(-1)
    gt = labels.numpy().reshape(-1).astype(np.int64)
    gt[gt == 255] = C
    ok = gt >= 0
    want = np.bincount((C + 1) * pred[ok] + gt[ok], minlength=(C + 1) ** 2).reshape(C + 1, C + 1)
    assert np.array_equal(conf.numpy(), want) and int(inv) == 4
    assert pred[0] == 3 and pred[H * W + 2 * W + 2] == 4


def test_evaluator_reports_invalid_labels(ref_backend):
    ev = SemSegEvaluator(4, ignore_label=255)
    t = torch.rand((4, 3, 5))
    ev.process([{"sem_seg": np.full((3, 5), 9, np.int64)}], [{"sem_seg": t}])
    with pytest.raises(ValueError, match="15 ground-truth pixels"):
        ev.evaluate()
    ev.reset()
    assert ev.evaluate()["sem_seg"]["mIoU"] is None  # nothing processed: NaN metrics, None as in the reference


def test_instance_configs_raise():
    proc = MaskFormerProcessor(MaskFormerConfig(num_classes=80, postprocessing_type="instance"))
    out = MaskFormerModelOutput(masks=LazyMasks(torch.zeros((1, 4, 4, 8)), 8, (16, 16)), logits=torch.zeros((1, 8, 80)))
    with pytest.raises(NotImplementedError, match="instance"):
        proc.eval_postprocess(out, [{"height": 16, "width": 16}])


def test_detection_eval_is_unchanged(ref_backend):
    """inference_on_dataset on a fai-detr model: the BoxAPEvaluator dict of the loop it has always run (model(x), eval_postprocess, process)"""
    from tests.test_api_cpu import _fm
    fm = _fm(size=128, num_classes=5)
    data = SyntheticDetectionDataset(n=3, size=128, num_classes=5)
    got = inference_on_dataset(fm, data, batch_size=2)
    ev = BoxAPEvaluator(5)
    for s in (0, 2):
        entries = [data[i] for i in range(s, min(3, s + 2))]
        out = fm.model(torch.stack([e["image"] for e in entries]).float())
        ev.process(entries, fm.processor.eval_postprocess(out, entries, None))
    assert got == ev.evaluate()


def test_synthetic_sem_seg_dataset():
    ds = SyntheticSemSegDataset(n=4, sizes=((357, 483), (250, 333)), seed=3)
    e0, e3 = ds[0], ds[3]
    assert tuple(e0["image"].shape) == (3, 357, 483) and e0["image"].dtype == torch.uint8 and (e0["height"], e0["width"]) == (357, 483)
    assert tuple(e3["sem_seg"].shape) == (250, 333) and tuple(ds[1]["image"].shape) == (3, 357, 483)
    gt = e0["sem_seg"]
    assert gt.dtype == torch.uint8 and 0.02 < float((gt == 255).float().mean()) < 0.08 and int(gt[gt != 255].max()) < 150
    assert torch.equal(ds[2]["sem_seg"], SyntheticSemSegDataset(n=4, sizes=((357, 483), (250, 333)), seed=3)[2]["sem_seg"])
