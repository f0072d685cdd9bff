"""Host-side orchestration of MaskFormer and BisenetFormer at image sizes that are not multiples of 32 (odd feature maps, non-x2 upsamples), on the CPU
operator references, against golden fixtures produced by the unmodified reference (oracle/gen_golden_any_size.py)."""
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import DETRConfig, FAIDetr, ops
from focoos_b200.bisenetformer import BisenetFormer, BisenetFormerConfig
from focoos_b200.fai_mf import FAIMaskFormer, MaskFormerConfig
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import state_dict_digest, synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import GOLDEN, load_golden, manifest_template

FAMILIES = {"mf_l_coco_ins": (FAIMaskFormer, MaskFormerConfig, "fai_mf_l_coco_ins"),
            "bisenetformer_l_ade": (BisenetFormer, BisenetFormerConfig, "bisenetformer_l_ade")}


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


def _meta():
    with open(os.path.join(GOLDEN, "golden_meta_any_size.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
@pytest.mark.parametrize("name", ["mf_l_coco_ins_b2_357x483", "mf_l_coco_ins_b1_720x1280", "bisenetformer_l_ade_b2_357x483", "bisenetformer_l_ade_b1_720x1280"])
def test_host_graph_matches_golden_at_any_size(ref_backend, name, precision):
    meta = _meta()[name]
    g = load_golden(name)
    cls, cfg, manifest = FAMILIES[name.split("_b")[0]]
    sd = seeded_state_dict(manifest_template(manifest), 0)
    assert state_dict_digest(sd) == meta["weights_sha256"]
    m = cls(cfg(), precision=precision)
    m.load_state_dict(sd, strict=True)
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    out = m(x, taps=taps)
    assert tuple(out.masks.shape[-2:]) == tuple(g["sizes"][0])
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2)[:, ::10, ::2, ::2].float().numpy()
    assert pm.shape == g["pred_masks_q10_s2"].shape
    # pre-sigmoid mask logits relative to their scale (|logit| ~ 1e2 with the seeded weights), as in the golden tests at multiples of 32
    e_logit = float(np.abs(pm - g["pred_masks_q10_s2"]).max())
    e_cls = float(np.abs(out.logits.numpy() - g["logits"]).max())
    e_mask = float(np.abs(out.masks[:, ::10, ::4, ::4].numpy() - g["masks_q10_s4"]).max())
    tol = 1e-3 if precision == "fp32" or name.startswith("bisenet") else 2e-3
    assert e_logit <= (1e-4 if precision == "fp32" else 1e-3) * scale and e_cls <= tol and e_mask <= tol, (e_logit, e_cls, e_mask)
    dets = MaskFormerProcessor(m.config).postprocess(out, imgs, threshold=float(g["threshold"]))
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        if n:
            assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() < 1e-3
            if precision == "fp32":
                assert [x.bbox for x in d.detections] == g["det_boxes"][i, :n].tolist()


def test_detr_still_requires_multiples_of_32(ref_backend):
    """DETRProcessor resizes to im_size; the engine keeps rejecting other sizes with a clear message"""
    with pytest.raises(ValueError, match="multiple of 32"):
        FAIDetr(DETRConfig())(torch.zeros(1, 3, 100, 128))
