"""Host-side orchestration of the MaskFormer family on a GPU-less machine (reference ops backend), against golden fixtures
produced by the unmodified reference (oracle/gen_golden_mf.py)."""
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import ops
from focoos_b200.fai_mf import FAIMaskFormer, MaskFormerConfig, MaskFormerModelOutput
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import state_dict_digest, synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import GOLDEN, ConvCalls, load_golden, manifest_template


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


def _sd():
    return seeded_state_dict(manifest_template("fai_mf_l_coco_ins"), 0)


def test_mf_state_dict_keys_match_reference_manifest():
    m = FAIMaskFormer(MaskFormerConfig())
    own = {k: (tuple(v.shape), v.dtype) for k, v in m.state_dict().items()}
    ref = {k: (tuple(v.shape), v.dtype) for k, v in manifest_template("fai_mf_l_coco_ins").items()}
    assert own.keys() == ref.keys(), sorted(set(own) ^ set(ref))[:10]
    assert own == ref


def test_mf_fused_graph_matches_golden(ref_backend):
    g = load_golden("mf_l_coco_ins_b2_320x416")
    with open(os.path.join(GOLDEN, "golden_meta_mf.json")) as f:
        meta = json.load(f)
    sd = _sd()
    assert state_dict_digest(sd) == meta["weights_sha256"]
    m = FAIMaskFormer(MaskFormerConfig(), precision="fp32")
    m.load_state_dict(sd, strict=True)
    imgs = synth_images(3, [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    out = m(x, taps=taps)
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2)  # NHWC -> [B,Q,h,w]
    # pre-sigmoid mask logits: with the seeded weights they reach |133|, so the 1e-3-abs bar (meant for O(10) logits) is applied
    # relative to that scale: 1e-4 * max|logit|  (fp32 reassociation between two fp32 implementations is ~3e-5 relative)
    assert np.abs(pm[:, ::4].numpy() - g["pred_masks_q4"]).max() <= 1e-4 * scale, "pre-sigmoid mask logits"
    assert np.abs(out.logits.numpy() - g["logits"]).max() <= 1e-3
    assert np.abs(out.masks[:, ::10, ::4, ::4].numpy() - g["masks_q10_s4"]).max() <= 1e-3
    proc = MaskFormerProcessor(m.config)
    dets = proc.postprocess(out, imgs, threshold=float(g["threshold"]))
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() < 1e-4
        assert [x.bbox for x in d.detections] == g["det_boxes"][i, :n].tolist()
    # the lazy path (what FocoosModel.__call__ uses): statistics from the low-resolution logits, only the kept masks upsampled - same detections
    m.lazy_masks = True
    lazy_out = m(x)
    m.lazy_masks = False
    assert hasattr(lazy_out.masks, "materialize")
    dets2 = proc.postprocess(lazy_out, imgs, threshold=float(g["threshold"]))
    for a_, b_ in zip(dets, dets2):
        assert [(d.cls_id, d.bbox, d.mask) for d in a_.detections] == [(d.cls_id, d.bbox, d.mask) for d in b_.detections]
        assert np.allclose([d.conf for d in a_.detections], [d.conf for d in b_.detections], rtol=1e-6)


def test_mf_pair_backbone_runs_as_pair_convs(ref_backend):
    """precision="fp32_tc": the ResNet backbone runs in the pair format (fp16 hi/lo planes between convs, ResNetTrunk.run) and the four pixel-decoder
    convs read the pairs - host-side bookkeeping on the CPU references: same outputs as the fp32 graph up to the pair rounding (2^-22 relative per activation)."""
    g = load_golden("mf_l_coco_ins_b2_320x416")
    m = FAIMaskFormer(MaskFormerConfig(), precision="fp32_tc")
    m.load_state_dict(_sd(), strict=True)
    imgs = synth_images(3, [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    ops._backend = calls = ConvCalls(ops._backend)
    out = m(x, taps=taps)
    eng = m.engine()
    backbone = [eng.trunk.stem2, eng.trunk.stem3] + [blk[k] for st in eng.trunk.stages for blk in st for k in ("a", "b", "c", "short") if blk[k] is not None]
    paired = {id(w) for w in calls.w["conv2d_pair"]}
    assert all(id(c.w3) in paired for c in backbone + [eng.pd_in, *eng.adapter.values(), eng.layer[1], eng.mask_features])
    assert not any(c.w is w or c.w3 is w for c in backbone for w in calls.w["conv2d"])
    assert np.abs(out.logits.numpy() - g["logits"]).max() <= 1e-3
    assert np.abs(out.masks[:, ::10, ::4, ::4].numpy() - g["masks_q10_s4"]).max() <= 2e-3
