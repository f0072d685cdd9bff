"""Generate the fai-detr-m-coco fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (STDC-2 trunk, no AIFI layer, 3 decoder layers).

TEST INFRASTRUCTURE.  Run in the build container only (needs the reference tree):

    python -m oracle.gen_golden_detr_m

Same recipe as oracle/gen_golden.py: the reference `ModelManager.get` model with the seeded weights (seed 0), run on CPU through its own
`processor.preprocess -> model.forward -> processor.postprocess` on seeded synthetic images (seed 1, 2 x 640x640, threshold 0.5), with forward hooks
on the STDC stage ends, the FPN / PAN blocks, the decoder layers and the last score head, and the encoder top-k recorded.
"""
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
from oracle.gen_golden import GOLDEN, TopkRecorder, state_dict_digest, synth_images  # noqa: E402

NAME, TAG = "fai-detr-m-coco", "detr_m_coco_b2_640"
HOOKS = {
    "pixel_decoder.backbone.features.5": "res3",
    "pixel_decoder.backbone.features.10": "res4",
    "pixel_decoder.backbone.features.13": "res5",
    "pixel_decoder.fpn_blocks.0": "fpn0",
    "pixel_decoder.fpn_blocks.1": "fpn1",
    "pixel_decoder.pan_blocks.0": "pan0",
    "pixel_decoder.pan_blocks.1": "pan1",
    "head.predictor.enc_output": "output_memory",
    "head.predictor.decoder.layers.0": "dec0_out",
    "head.predictor.decoder.layers.2": "dec2_out",
    "head.predictor.dec_score_classifier.2": "pred_logits",
}


def main():
    fm = ref_import.get_reference_model(NAME)
    m, proc = fm.model, fm.processor
    template = m.state_dict()
    manifest = {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in template.items()}
    with open(os.path.join(GOLDEN, "fai_detr_m_coco_state_dict_manifest.json"), "w") as f:
        json.dump(manifest, f, indent=0, sort_keys=True)
    sd = seeded_state_dict(template, seed=0)
    m.load_state_dict(sd, strict=True)
    m.eval()

    taps, hs = {}, []
    mods = dict(m.named_modules())
    for n, t in HOOKS.items():
        hs.append(mods[n].register_forward_hook(lambda mod, inp, out, t=t: taps.__setitem__(t, out.detach().clone())))
    images, threshold = synth_images(1, [(640, 640)] * 2), 0.5
    with torch.no_grad(), TopkRecorder() as rec:
        x, _ = proc.preprocess(images, device=torch.device("cpu"), dtype=torch.float32)
        out = m(x)
        dets = proc.postprocess(out, images, class_names=[], threshold=threshold)
    for h in hs:
        h.remove()
    B = x.shape[0]
    enc_topk = [c for c in rec.calls if c[0] == (B, 8400)]
    post_topk = [c for c in rec.calls if c[0] == (300 * out.logits.shape[-1],)]
    assert len(enc_topk) == 1 and len(post_topk) == B
    g = {
        "scores": out.logits.numpy(),
        "boxes": out.boxes.numpy(),
        "enc_topk_ind": enc_topk[0][1].numpy().astype(np.int32),
        "enc_topk_val": enc_topk[0][2].numpy(),
        "post_topk_ind": np.stack([c[1].numpy() for c in post_topk]).astype(np.int32),
        "pre_image_mean": x.mean(dim=(2, 3)).numpy(),
        "pre_image_patch": x[:, :, 100:108, 200:208].numpy(),
        "det_count": np.array([len(d.detections) for d in dets], dtype=np.int32),
        "image_sizes": np.array([im.shape[:2] for im in images], dtype=np.int32),
        "threshold": np.float32(threshold),
    }
    nmax = max(1, int(g["det_count"].max()))
    db, ds, dl = np.zeros((B, nmax, 4), np.int32), np.zeros((B, nmax), np.float32), np.full((B, nmax), -1, np.int32)
    for i, d in enumerate(dets):
        for j, det in enumerate(d.detections):
            db[i, j], ds[i, j], dl[i, j] = det.bbox, det.conf, det.cls_id
    g.update(det_boxes=db, det_scores=ds, det_labels=dl)
    for t in ("res3", "res4", "res5", "fpn0", "fpn1", "pan0", "pan1"):  # channel-sliced, NCHW as the reference lays them out
        v = taps[t]
        g["tap_" + t] = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        g["tapstat_" + t] = np.array([v.mean().item(), v.std().item(), v.abs().max().item()], np.float32)
    g["tap_output_memory"] = taps["output_memory"][:, ::97, ::4].numpy()
    g["tap_dec0_out"] = taps["dec0_out"][:, :, ::8].numpy()
    g["tap_dec2_out"] = taps["dec2_out"][:, :, ::8].numpy()
    g["pred_logits_raw"] = taps["pred_logits"].numpy()
    np.savez_compressed(os.path.join(GOLDEN, TAG + ".npz"), **g)

    meta = {"model": NAME, "weights_seed": 0, "weights_sha256": state_dict_digest(sd), "torch": torch.__version__, "reference_version": "0.25.0",
            "cases": {TAG: {"image_seed": 1, "sizes": [[640, 640]] * 2, "threshold": threshold, "det_count": g["det_count"].tolist()}}}
    with open(os.path.join(GOLDEN, "golden_meta_detr_m.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print(json.dumps(meta, indent=1))


if __name__ == "__main__":
    main()
