"""Semantic evaluation on the GPU: the confusion kernel against fp64 argmax + bincount; eval_postprocess against the reference's einsum and labels / metrics
against the UNMODIFIED reference's goldens (tests/golden/sem_seg_eval_*.npz); model.eval of the five ADE20K semantic models in fp32 and fp32_tc."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import ModelManager, ops
from focoos_b200.fai_mf import LazyMasks, MaskFormerModelOutput
from focoos_b200.trainer import SemSegEvaluator, SyntheticSemSegDataset, TrainerArgs, inference_on_dataset
from focoos_b200.utils.seeded_weights import seeded_state_dict
from tests.test_sem_seg_eval_cpu import GOLDEN, MODEL_CASES, _case, _model_case, _proc, golden_metrics

pytestmark = pytest.mark.gpu

# product bars, relative to max |sem_seg|: fp32 (CUDA-core fp32) and fp32_tc (three fp16 tensor-core products on hi / lo halves, ~2^-21 per product)
REL = {"fp32": 1e-5, "fp32_tc": 1e-5}
# labels are compared where the reference's top-2 margin exceeds EPS * max |sem_seg|: the processor case differs from the reference only by fp32 rounding;
# the seeded model decoders amplify a 1e-6 input perturbation to ~3e-3 in the class probabilities (DESIGN §2), so the model cases take a wider margin; on the
# seeded fai-mf-m-ade the scores of most pixels lie within it (about 309k of 369k pixels), so its label and metric checks are weak - bisenetformer-s-ade has none
EPS_PROC, EPS_MODEL = 1e-4, 2e-2


def _ref_confusion(scores, labels, C, ignore):
    pred = torch.argmax(scores[..., :C].double().cpu(), -1).reshape(-1).numpy()
    gt = labels.cpu().numpy().reshape(-1).astype(np.int64)
    gt[gt == ignore] = C
    ok = (gt >= 0) & (gt <= C)
    return np.bincount((C + 1) * pred[ok] + gt[ok], minlength=(C + 1) ** 2).reshape(C + 1, C + 1), int((~ok).sum())


@pytest.mark.parametrize("B,H,W,Cp,dtype", [(1, 1, 1, 152, torch.uint8), (16, 37, 53, 152, torch.uint8), (16, 40, 31, 256, torch.int32), (1, 1080, 1920, 152, torch.uint8),
                                            (2, 64, 96, 1032, torch.int32)])  # the last: C = 1031, direct global adds (no shared histogram)
def test_confusion_kernel_matches_fp64_argmax_bincount(B, H, W, Cp, dtype):
    C = 150 if Cp < 1000 else 1031
    g = torch.Generator().manual_seed(B * 7 + H)
    scores = torch.randint(0, 6, (B, H, W, Cp), generator=g).float()  # small integer values: many exact ties at the maximum
    scores += torch.rand(scores.shape, generator=g) * (torch.rand(scores.shape, generator=g) < 0.5)
    scores[..., C:] = 1e9  # padding channels never count
    flat = scores.view(-1, Cp)
    n = flat.shape[0]
    flat[::7, 3] = float("nan")
    flat[::11, [5, 9]] = float("nan")
    flat[::13, :C] = float("-inf")
    labels = torch.randint(0, C, (B, H, W), generator=g).to(dtype)
    labels.view(-1)[::17] = 255 if dtype == torch.uint8 or C < 255 else -1
    if B > 1:
        labels[1] = 255  # an all-ignore image
    if dtype == torch.int32:
        labels.view(-1)[::29] = C  # counted in the ignore column, as bincount does
    want, want_bad = _ref_confusion(scores, labels, C, 255)
    sd, ld = scores.cuda(), labels.cuda()
    runs = []
    for _ in range(2):
        conf = torch.zeros((C + 1, C + 1), dtype=torch.int64, device="cuda")
        bad = torch.zeros((1,), dtype=torch.int64, device="cuda")
        ops.sem_seg_confusion(sd, ld, C, 255, conf, bad)
        runs.append((conf.cpu().numpy(), int(bad)))
    assert np.array_equal(runs[0][0], want) and runs[0][1] == want_bad
    assert np.array_equal(runs[1][0], runs[0][0]) and int(runs[0][0].sum()) == n - want_bad


def test_confusion_kernel_reads_a_channel_slice():
    g = torch.Generator().manual_seed(5)
    buf = torch.rand((3, 20, 30, 160), generator=g)
    labels = torch.randint(0, 151, (3, 20, 30), generator=g, dtype=torch.int32)
    want, _ = _ref_confusion(buf[..., 4:154], labels, 150, 255)
    conf = torch.zeros((151, 151), dtype=torch.int64, device="cuda")
    bad = torch.zeros((1,), dtype=torch.int64, device="cuda")
    ops.sem_seg_confusion(buf.cuda()[..., 4:154], labels.cuda(), 150, 255, conf, bad)
    assert np.array_equal(conf.cpu().numpy(), want)


def _near_ties(z, i, pred, eps):
    m = z[f"margin_{i}"].astype(np.float32)
    far = m > eps
    return int((~far).sum()), bool(np.array_equal(pred[far], z[f"pred_{i}"][far]))


def _metrics_within(got, want, n_near, conf):
    """each near-tie pixel moves one count between two classes: a per-class IoU / ACC moves by at most 1 / (its smallest non-zero union), pACC by 1 / pixels"""
    if n_near == 0:
        assert got == want
        return
    pos = np.concatenate([conf[:-1, :-1].sum(0), conf[:-1, :-1].sum(1)])
    bound = 100.0 * 2 * n_near / max(1, int(pos[pos > 0].min()))
    for k in ("mIoU", "fwIoU", "mACC", "pACC"):
        assert abs(got[k] - want[k]) <= bound, (k, got[k], want[k], bound)


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16"])
def test_eval_postprocess_matches_the_reference(precision):
    low, logits, entries, gts = _case()
    Q, (H, W) = logits.shape[1], entries[0]["image_size"]
    # the NHWC probabilities hold the values of LazyMasks.materialize()
    p_nhwc = ops.mask_sigmoid_upsample_nhwc(low.cuda(), Q, (H, W), 128, "fp32")
    p_mat = ops.mask_sigmoid_upsample(low.cuda(), Q, (H, W)).permute(0, 2, 3, 1)
    assert float((p_nhwc[..., :Q] - p_mat).abs().max()) <= 1e-7 and not p_nhwc[..., Q:].any()
    out = _proc().eval_postprocess(MaskFormerModelOutput(masks=LazyMasks(low.cuda(), Q, (H, W)), logits=logits.cuda()), entries, precision=precision)
    probs = F.interpolate(torch.sigmoid(low.permute(0, 3, 1, 2)[:, :Q]), size=(H, W), mode="bilinear", align_corners=False)
    z = np.load(os.path.join(GOLDEN, "sem_seg_eval_proc.npz"))
    near = 0
    for i, (o, e) in enumerate(zip(out, entries)):
        p = probs[i:i + 1] if (e["height"], e["width"]) == (H, W) else F.interpolate(probs[i:i + 1], size=(e["height"], e["width"]), mode="bilinear", align_corners=False)
        ref = torch.einsum("qc,qhw->chw", logits[i].double(), p[0].double())
        t = o["sem_seg"].double().cpu()
        rel = float((t - ref).abs().max() / ref.abs().max())
        assert rel <= REL.get(precision, 1e-2), (precision, i, rel)
        n, same = _near_ties(z, i, t.argmax(0).numpy(), EPS_PROC * float(ref.abs().max()))
        near += n
        if precision != "fp16":
            assert same, (precision, i)
    print(f"[sem_seg] eval_postprocess {precision}: near-tie pixels {near}")
    if precision != "fp16":
        ev = SemSegEvaluator(150)
        ev.process([{"sem_seg": gt} for gt in gts], out)
        conf = ev.confusion_matrix()
        assert np.abs(conf - z["conf"]).sum() <= 2 * near
        _metrics_within(ev.evaluate()["sem_seg"], golden_metrics(z), near, z["conf"])


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
@pytest.mark.parametrize("name", MODEL_CASES)
def test_model_eval_matches_the_reference(name, precision):
    z = np.load(os.path.join(GOLDEN, "sem_seg_eval_" + name.replace("-", "_") + ".npz"))
    with open(os.path.join(GOLDEN, name.replace("-", "_") + "_state_dict_manifest.json")) as f:
        man = json.load(f)
    sd = seeded_state_dict({k: torch.empty(v[0], dtype=getattr(torch, v[1])) for k, v in man.items()}, 0)
    fm = ModelManager.get(name, state_dict=sd, precision=precision)
    imgs, entries, gts = _model_case()
    data = [{"image": torch.from_numpy(im).permute(2, 0, 1).contiguous(), "height": e["height"], "width": e["width"], "sem_seg": gt}
            for im, e, gt in zip(imgs, entries, gts)]
    got = inference_on_dataset(fm, data, batch_size=16)["sem_seg"]
    near = 0
    for idx in ([0, 1], [2]):  # the batches inference_on_dataset formed
        x = torch.stack([data[i]["image"] for i in idx]).cuda().float()
        fm.model.lazy_masks = True
        out = fm.model(x)
        fm.model.lazy_masks = False
        res = fm.processor.eval_postprocess(out, [data[i] for i in idx], precision=precision)
        for i, r in zip(idx, res):
            t = r["sem_seg"]
            n, same = _near_ties(z, i, t.argmax(0).cpu().numpy(), EPS_MODEL * float(t.abs().max()))
            near += n
            assert same, (name, precision, i)
    print(f"[sem_seg] {name} {precision}: near-tie pixels {near}, mIoU {got['mIoU']} (reference {golden_metrics(z)['mIoU']})")
    _metrics_within(got, golden_metrics(z), near, z["conf"])


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
@pytest.mark.parametrize("name", ["fai-mf-l-ade", "fai-mf-m-ade", "bisenetformer-l-ade", "bisenetformer-m-ade", "bisenetformer-s-ade"])
def test_model_eval_runs_on_the_ade_models(name, precision, tmp_path):
    fm = ModelManager.get(name, precision=precision)
    data = SyntheticSemSegDataset(n=4, sizes=((357, 483), (250, 333)))
    m = fm.eval(TrainerArgs(run_name="e", output_dir=str(tmp_path), batch_size=2), data, save_json=True)
    res = m["sem_seg"]
    assert list(res)[:2] == ["mIoU", "fwIoU"] and len(res) == 4 + 2 * 150 and res["pACC"] is not None
    assert 0.0 <= res["pACC"] <= 100.0 and os.path.exists(tmp_path / "e" / "eval_metrics.json")
