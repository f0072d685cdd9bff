"""Goldens for semantic evaluation FROM THE UNMODIFIED REFERENCE (needs the reference tree):  python -m oracle.gen_golden_sem_seg_eval

(a) tests/golden/sem_seg_eval_proc.npz: the reference's MaskFormerProcessor.eval_postprocess (models/fai_mf/processor.py:142-166) and SemSegEvaluator
    (trainer/evaluation/sem_seg_evaluation.py) alone, on the seeded case of tests/test_sem_seg_eval_cpu.py (`_case`): C = 150, Q = 100, exact and near
    ties between class columns, one entry whose (height, width) differs from the mask size, ground truth with ignore pixels.  The mask probabilities
    are the reference head's: sigmoid of the low-resolution logits, then F.interpolate to the input size (fai_mf/modelling.py:619,722-723).
(b) tests/golden/sem_seg_eval_<model>.npz: the reference model with the seeded state_dict (seed 0) for bisenetformer-s-ade and fai-mf-m-ade on two
    256x384 images (one batch) and one 357x483 image (`_model_case`), then the same processor and evaluator.
Each stores per image the reference's argmax map and its top-2 margin (fp16), the confusion matrix and the metrics (keys, values with NaN for None)."""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from focoos_b200.utils.seeded_weights import seeded_state_dict  # noqa: E402
from oracle import ref_import  # noqa: E402
from tests.test_sem_seg_eval_cpu import MODEL_CASES, _case, _model_case  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _reference_eval(proc, batches, entries, gts, num_classes):
    """the reference's eval_postprocess per batch ((indices, masks, logits)), then SemSegEvaluator.process / evaluate over all images -> the arrays of one golden"""
    from focoos.models.fai_mf.ports import MaskFormerModelOutput
    from focoos.trainer.evaluation.sem_seg_evaluation import SemSegEvaluator

    class Entry:  # DatasetEntry duck type
        def __init__(self, i, e):
            self.image = torch.zeros((3, *e["image_size"]))
            self.height, self.width = e["height"], e["width"]
            self.sem_seg_file_name = self.file_name = str(i)

    ents, outs = [], []
    for idx, masks, logits in batches:
        be = [Entry(i, entries[i]) for i in idx]
        ents += be
        outs += proc.eval_postprocess(MaskFormerModelOutput(masks=masks, logits=logits, loss=None), be)
    meta = SimpleNamespace(name="synthetic", ignore_label=255, stuff_classes=[str(i) for i in range(num_classes)])
    ev = SemSegEvaluator(SimpleNamespace(metadata=meta), distributed=False, sem_seg_loading_fn=lambda name, dtype: gts[int(name)].astype(dtype))
    ev.encode_json_sem_seg = lambda *a: []  # the JSON dump of predictions is not evaluated here
    ev.reset()
    ev.process(ents, outs)
    res = ev.evaluate()["sem_seg"]
    g = {"conf": ev._conf_matrix, "metric_keys": np.array(list(res)), "metric_vals": np.array([np.nan if v is None else v for v in res.values()], np.float64)}
    for i, o in enumerate(outs):
        t = o["sem_seg"]
        top2 = t.topk(2, dim=0).values
        g[f"pred_{i}"] = t.argmax(0).numpy().astype(np.uint8)
        g[f"margin_{i}"] = np.minimum((top2[0] - top2[1]).numpy(), 6e4).astype(np.float16)
    return g


def main():
    ref_import.install()
    from focoos.models.fai_mf.config import MaskFormerConfig as RC
    from focoos.models.fai_mf.processor import MaskFormerProcessor as RP
    from focoos.nn.backbone.resnet import ResnetConfig as RB

    low, logits, entries, gts = _case()
    H, W = entries[0]["image_size"]
    masks = F.interpolate(torch.sigmoid(low.permute(0, 3, 1, 2)[:, :logits.shape[1]]), size=(H, W), mode="bilinear", align_corners=False)
    proc = RP(RC(backbone_config=RB(), num_classes=150, postprocessing_type="semantic", predict_all_pixels=True, use_mask_score=False))
    g = _reference_eval(proc, [(list(range(len(entries))), masks, logits)], entries, gts, 150)
    np.savez_compressed(os.path.join(GOLDEN, "sem_seg_eval_proc.npz"), **g)
    print("proc", dict(zip(g["metric_keys"][:2], g["metric_vals"][:2])), flush=True)

    for name in MODEL_CASES:
        fm = ref_import.get_reference_model(name)
        fm.model.load_state_dict(seeded_state_dict(fm.model.state_dict(), seed=0), strict=True)
        fm.model.eval()
        imgs, entries, gts = _model_case()
        batches = []
        for idx in ([0, 1], [2]):  # the batches inference_on_dataset forms: consecutive entries of one image size
            x = torch.stack([torch.from_numpy(imgs[i]).permute(2, 0, 1).float() for i in idx])
            with torch.no_grad():
                out = fm.model(x)
            batches.append((idx, out.masks, out.logits))
        g = _reference_eval(fm.processor, batches, entries, gts, 150)
        np.savez_compressed(os.path.join(GOLDEN, "sem_seg_eval_" + name.replace("-", "_") + ".npz"), **g)
        print(name, dict(zip(g["metric_keys"][:2], g["metric_vals"][:2])), flush=True)


if __name__ == "__main__":
    main()
