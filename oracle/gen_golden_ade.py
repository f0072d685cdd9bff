"""Golden fixtures for the ADE20K semantic segmenters FROM THE UNMODIFIED REFERENCE (build container only):

    python -m oracle.gen_golden_ade

fai-mf-l-ade (R101-vd) and fai-mf-m-ade (STDC-2): 128-wide TransformerFPN without encoder layers (layer_4 reads res5), 6 / 3 masked decoder layers;
bisenetformer-m-ade (STDC-2, 96-wide pixel decoder, 4 decoder layers) and bisenetformer-s-ade (STDC-1, 128-wide).  Per model, with the seeded state_dict
(seed 0):
  * the state_dict manifest,
  * B=2 at 320x416 (fai-mf, image seed 3; 5 for fai-mf-l-ade) or 256x384 (bisenetformer, image seed 4): class probabilities, pre-sigmoid mask logits of every 10th query at every
    2nd low-resolution pixel, final mask probabilities of every 10th query at every 4th pixel (the sampling of gen_golden_any_size.py), a mask-feature tap
    and the reference's semantic detections,
and for fai-mf-m-ade and bisenetformer-m-ade one odd-size case, B=2 at 357x483 (image seed 5 / 9), without the tap and with the final probabilities of
every 20th query only (masks_q20_s4: every 10th query puts the fai-mf-m-ade file over 1 MB).
fai-mf-l-ade takes image seed 5: on seeds 3 and 4 the reference's semantic post-process keeps a one-pixel-wide mask, whose trimmed crop is empty, and
its PNG encoder raises."""
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
MODELS = ["fai-mf-l-ade", "fai-mf-m-ade", "bisenetformer-m-ade", "bisenetformer-s-ade"]
# (reference model, image seed, sizes, with the mask-feature tap)
CASES = [
    ("fai-mf-l-ade", 5, [(320, 416), (320, 416)], True),
    ("fai-mf-m-ade", 3, [(320, 416), (320, 416)], True),
    ("fai-mf-m-ade", 5, [(357, 483), (357, 483)], False),
    ("bisenetformer-m-ade", 4, [(256, 384), (256, 384)], True),
    ("bisenetformer-m-ade", 9, [(357, 483), (357, 483)], False),
    ("bisenetformer-s-ade", 4, [(256, 384), (256, 384)], True),
]


def tag(name):
    return name.replace("fai-", "").replace("-", "_")  # fai-mf-m-ade -> mf_m_ade, bisenetformer-s-ade -> bisenetformer_s_ade


def manifest_name(name):
    return name.replace("-", "_") + "_state_dict_manifest"  # fai_mf_m_ade_state_dict_manifest


def golden_name(name, sizes):
    return f"{tag(name)}_b{len(sizes)}_{sizes[0][0]}x{sizes[0][1]}"


def main():
    meta = {}
    models = {}
    for name in MODELS:
        fm = ref_import.get_reference_model(name)
        template = fm.model.state_dict()
        with open(os.path.join(GOLDEN, manifest_name(name) + ".json"), "w") as f:
            json.dump({k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in template.items()}, f, indent=0, sort_keys=True)
        sd = seeded_state_dict(template, seed=0)
        fm.model.load_state_dict(sd, strict=True)
        fm.model.eval()
        models[name] = (fm, state_dict_digest(sd))
        print(name, len(template), "keys", flush=True)
    from focoos.models.fai_mf.ports import MaskFormerModelOutput

    for name, seed, sizes, with_tap in CASES:
        fm, digest = models[name]
        imgs = synth_images(seed, sizes)
        x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
        taps = {}
        # both families' pixel decoders return (mask_features, multi-scale features)
        hooks = [fm.model.head.predictor.register_forward_hook(lambda m, i, o: taps.__setitem__("pred", {k: v.detach() for k, v in o.items() if k != "aux_outputs"})),
                 fm.model.pixel_decoder.register_forward_hook(lambda m, i, o: taps.__setitem__("mask_features", o[0].detach()))]
        with torch.no_grad():
            out = fm.model(x)
        for h in hooks:
            h.remove()
        pm = taps["pred"]["pred_masks"]
        g = {
            "logits": out.logits.numpy(),                                           # [B,Q,K] softmax probs without no-object
            "pred_masks_stat": np.array([pm.mean().item(), pm.std().item(), pm.abs().max().item()], np.float32),
            "pred_masks_q10_s2": pm[:, ::10, ::2, ::2].numpy(),                     # pre-sigmoid, every 10th query, every 2nd low-resolution pixel
            "sizes": np.array(sizes, np.int32),
        }
        if with_tap:
            g["masks_q10_s4"] = out.masks[:, ::10, ::4, ::4].numpy()                # final probabilities, subsampled
            g["mask_features_tap"] = taps["mask_features"][:, ::16, ::4, ::4].numpy()
        else:
            g["masks_q20_s4"] = out.masks[:, ::20, ::4, ::4].numpy()
        g.update(_detections(fm, out, imgs, MaskFormerModelOutput))
        fname = golden_name(name, sizes)
        np.savez_compressed(os.path.join(GOLDEN, fname + ".npz"), **g)
        meta[fname] = {"model": name, "weights_seed": 0, "weights_sha256": digest, "image_seed": seed, "sizes": [list(s) for s in sizes], "threshold": THR,
                       "det_count": g["det_count"].tolist(), "pred_masks_shape": list(pm.shape)}
        print(fname, meta[fname], "pred_masks stat", g["pred_masks_stat"], "max prob", out.logits.max().item(), flush=True)
    with open(os.path.join(GOLDEN, "golden_meta_ade.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
