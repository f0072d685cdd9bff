"""Golden fixtures for MaskFormer and BisenetFormer at image sizes that are not multiples of 32, FROM THE UNMODIFIED REFERENCE (build container only):

    python -m oracle.gen_golden_any_size

Same seeded state_dicts and taps as gen_golden_mf.py / gen_golden_bisenet.py.  Two inputs per family:
  * B=2 at 357x483: both dims odd.  ResNet maps 179x242 -> 90x121 -> 45x61 -> 23x31 -> 12x16 (stride-2 convs on an odd W and on maps with both dims odd,
    the ceil-mode average pool on odd maps, FPN nearest upsamples 12->23->45->90, a non-integer final mask upsample); STDC gives the same map chain.
  * B=1 at 720x1280: the last stride-2 layers run on 45x80."""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from focoos_b200.utils.seeded_weights import seeded_state_dict  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle.gen_golden import state_dict_digest, synth_images  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
THR = 0.5
# (family tag, reference model, image seed, sizes)
CASES = [
    ("mf_l_coco_ins", "fai-mf-l-coco-ins", 5, [(357, 483), (357, 483)]),
    ("mf_l_coco_ins", "fai-mf-l-coco-ins", 6, [(720, 1280)]),
    ("bisenetformer_l_ade", "bisenetformer-l-ade", 9, [(357, 483), (357, 483)]),
    ("bisenetformer_l_ade", "bisenetformer-l-ade", 8, [(720, 1280)]),
]


def golden_name(tag, sizes):
    return f"{tag}_b{len(sizes)}_{sizes[0][0]}x{sizes[0][1]}"


def _detections(fm, out, imgs, output_cls):
    ks, kl, kb = [], [], []
    for i in range(len(imgs)):
        o1 = output_cls(masks=out.masks[i:i + 1], logits=out.logits[i:i + 1], loss=None)
        dets = fm.processor.postprocess(o1, [imgs[i]], class_names=[], threshold=THR)[0]
        ks.append([d.conf for d in dets.detections]); kl.append([d.cls_id for d in dets.detections]); kb.append([d.bbox for d in dets.detections])
    n = max(1, max(len(s) for s in ks))
    ds = np.zeros((len(imgs), n), np.float32); dl = np.full((len(imgs), n), -1, np.int32); db = np.zeros((len(imgs), n, 4), np.int32); dc = np.zeros(len(imgs), np.int32)
    for i in range(len(imgs)):
        k = len(ks[i]); dc[i] = k; ds[i, :k] = ks[i]; dl[i, :k] = kl[i]
        if k:
            db[i, :k] = np.array(kb[i])
    return dict(det_scores=ds, det_labels=dl, det_boxes=db, det_count=dc, threshold=np.float32(THR))


def main():
    meta = {}
    models = {}
    for tag, name, seed, sizes in CASES:
        if name not in models:
            fm = ref_import.get_reference_model(name)
            sd = seeded_state_dict(fm.model.state_dict(), seed=0)
            fm.model.load_state_dict(sd, strict=True)
            fm.model.eval()
            models[name] = (fm, state_dict_digest(sd))
        fm, digest = models[name]
        imgs = synth_images(seed, sizes)
        x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
        taps = {}
        hooks = [fm.model.head.predictor.register_forward_hook(lambda m, i, o: taps.__setitem__("pred", {k: v.detach() for k, v in o.items() if k != "aux_outputs"}))]
        with torch.no_grad():
            out = fm.model(x)
        for h in hooks:
            h.remove()
        pm = taps["pred"]["pred_masks"]
        g = {
            "logits": out.logits.numpy(),                                       # [B,Q,K] class probabilities
            "pred_masks_q10_s2": pm[:, ::10, ::2, ::2].numpy(),                 # pre-sigmoid mask logits, every 10th query, every 2nd low-resolution pixel
            "pred_masks_stat": np.array([pm.mean().item(), pm.std().item(), pm.abs().max().item()], np.float32),
            "masks_q10_s4": out.masks[:, ::10, ::4, ::4].numpy(),               # final probabilities at the input size, subsampled
            "sizes": np.array(sizes, np.int32),
        }
        if tag.startswith("mf"):
            from focoos.models.fai_mf.ports import MaskFormerModelOutput as OutCls
        else:
            from focoos.models.bisenetformer.ports import BisenetFormerOutput as OutCls
        g.update(_detections(fm, out, imgs, OutCls))
        fname = golden_name(tag, sizes)
        np.savez_compressed(os.path.join(GOLDEN, fname + ".npz"), **g)
        meta[fname] = {"model": name, "weights_seed": 0, "weights_sha256": digest, "image_seed": seed, "sizes": [list(s) for s in sizes], "threshold": THR,
                       "det_count": g["det_count"].tolist(), "pred_masks_shape": list(pm.shape)}
        print(fname, meta[fname], "pred_masks stat", g["pred_masks_stat"], flush=True)
    with open(os.path.join(GOLDEN, "golden_meta_any_size.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
