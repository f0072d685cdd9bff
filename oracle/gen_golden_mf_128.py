"""Golden fixtures for the 128-wide MaskFormer pixel decoders FROM THE UNMODIFIED REFERENCE (build container only):

    python -m oracle.gen_golden_mf_128

fai-mf-m-coco-ins (R101-vd) and fai-mf-s-coco-ins (R50-vd): 128-channel TransformerFPN with 3 pre-norm encoder layers of 8 heads x 16 channels,
6 masked decoder layers of hidden 256, 128-wide mask features, instance post-processing.  Per model, with the seeded state_dict (seed 0):
  * the state_dict manifest,
  * B=2 at 320x416 (image seed 3): class probabilities, pre-sigmoid mask logits of every 10th query at every 2nd low-resolution pixel, final mask
    probabilities of every 10th query at every 4th pixel (the sampling of gen_golden_any_size.py, which keeps each file under 1 MB), encoder-memory and
    mask-feature taps, and the reference's post-processed detections,
and for fai-mf-s-coco-ins one odd-size case, B=2 at 357x483 (image seed 5), without the two taps."""
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
from oracle.gen_golden_any_size import _detections  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
THR = 0.5
MODELS = ["fai-mf-m-coco-ins", "fai-mf-s-coco-ins"]
# (reference model, image seed, sizes, tap set)
CASES = [
    ("fai-mf-m-coco-ins", 3, [(320, 416), (320, 416)], "full"),
    ("fai-mf-s-coco-ins", 3, [(320, 416), (320, 416)], "full"),
    ("fai-mf-s-coco-ins", 5, [(357, 483), (357, 483)], "any_size"),
]


def tag(name):
    return name.replace("fai-", "").replace("-", "_")  # fai-mf-s-coco-ins -> mf_s_coco_ins


def golden_name(name, sizes):
    return f"{tag(name)}_b{len(sizes)}_{sizes[0][0]}x{sizes[0][1]}"


def main():
    meta = {}
    models = {}
    for name in MODELS:
        fm = ref_import.get_reference_model(name)
        template = fm.model.state_dict()
        with open(os.path.join(GOLDEN, f"fai_{tag(name)}_state_dict_manifest.json"), "w") as f:
            json.dump({k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in template.items()}, f, indent=0, sort_keys=True)
        sd = seeded_state_dict(template, seed=0)
        fm.model.load_state_dict(sd, strict=True)
        fm.model.eval()
        models[name] = (fm, state_dict_digest(sd))
    from focoos.models.fai_mf.ports import MaskFormerModelOutput

    for name, seed, sizes, kind in CASES:
        fm, digest = models[name]
        imgs = synth_images(seed, sizes)
        x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
        taps = {}
        hooks = [fm.model.head.predictor.register_forward_hook(lambda m, i, o: taps.__setitem__("pred", {k: v.detach() for k, v in o.items() if k != "aux_outputs"}))]
        if kind == "full":
            hooks += [
                fm.model.pixel_decoder.mask_features.register_forward_hook(lambda m, i, o: taps.__setitem__("mask_features", o.detach())),
                fm.model.pixel_decoder.transformer.register_forward_hook(lambda m, i, o: taps.__setitem__("enc_memory", o.detach())),
            ]
        with torch.no_grad():
            out = fm.model(x)
        for h in hooks:
            h.remove()
        pm = taps["pred"]["pred_masks"]
        g = {
            "logits": out.logits.numpy(),                                           # [B,Q,K] softmax probs without no-object
            "pred_masks_stat": np.array([pm.mean().item(), pm.std().item(), pm.abs().max().item()], np.float32),
            "pred_masks_q10_s2": pm[:, ::10, ::2, ::2].numpy(),                     # pre-sigmoid, every 10th query, every 2nd low-resolution pixel
            "masks_q10_s4": out.masks[:, ::10, ::4, ::4].numpy(),                   # final probabilities, subsampled
            "sizes": np.array(sizes, np.int32),
        }
        if kind == "full":
            g.update(mask_features_tap=taps["mask_features"][:, ::32, ::4, ::4].numpy(), enc_memory_tap=taps["enc_memory"][:, ::32].numpy())
        g.update(_detections(fm, out, imgs, MaskFormerModelOutput))
        fname = golden_name(name, sizes)
        np.savez_compressed(os.path.join(GOLDEN, fname + ".npz"), **g)
        meta[fname] = {"model": name, "weights_seed": 0, "weights_sha256": digest, "image_seed": seed, "sizes": [list(s) for s in sizes], "threshold": THR,
                       "det_count": g["det_count"].tolist(), "pred_masks_shape": list(pm.shape)}
        print(fname, meta[fname], "pred_masks stat", g["pred_masks_stat"], "max prob", out.logits.max().item(), flush=True)
    with open(os.path.join(GOLDEN, "golden_meta_mf_128.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
