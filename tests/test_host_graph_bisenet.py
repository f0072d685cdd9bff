"""Host-side orchestration of the BisenetFormer family on a GPU-less machine (reference ops backend) vs reference goldens."""
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import ops
from focoos_b200.bisenetformer import BisenetFormer, BisenetFormerConfig
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


def test_bisenet_state_dict_keys_match_reference_manifest():
    m = BisenetFormer(BisenetFormerConfig())
    own = {k: (tuple(v.shape), v.dtype) for k, v in m.state_dict().items()}
    ref = {k: (tuple(v.shape), v.dtype) for k, v in manifest_template("bisenetformer_l_ade").items()}
    assert own.keys() == ref.keys(), sorted(set(own) ^ set(ref))[:10]
    assert own == ref


def test_bisenet_fused_graph_matches_golden(ref_backend):
    g = load_golden("bisenetformer_l_ade_b2_256x384")
    with open(os.path.join(GOLDEN, "golden_meta_bisenet.json")) as f:
        meta = json.load(f)
    sd = seeded_state_dict(manifest_template("bisenetformer_l_ade"), 0)
    assert state_dict_digest(sd) == meta["weights_sha256"]
    m = BisenetFormer(BisenetFormerConfig(), precision="fp32")
    m.load_state_dict(sd, strict=True)
    imgs = synth_images(4, [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    out = m(x, taps=taps)
    scale = float(g["pred_masks_stat"][2])
    assert np.abs(taps["cp32"].permute(0, 3, 1, 2)[:, ::16].numpy() - g["cp32_tap"]).max() <= 1e-4 * np.abs(g["cp32_tap"]).max()
    assert np.abs(taps["mask_features"].permute(0, 3, 1, 2)[:, ::16, ::2, ::2].numpy() - g["mask_features_tap"]).max() <= 1e-4 * np.abs(g["mask_features_tap"]).max()
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2)
    assert np.abs(pm[:, ::4].numpy() - g["pred_masks_q4"]).max() <= 1e-4 * scale
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
    # the lazy path (what FocoosModel.__call__ uses): semantic argmax straight from the low-resolution logits - same detections
    m.lazy_masks = True
    lazy_out = m(x)
    m.lazy_masks = False
    assert hasattr(lazy_out.masks, "materialize") and tuple(lazy_out.masks.shape) == tuple(out.masks.shape)
    dets2 = proc.postprocess(lazy_out, imgs, threshold=float(g["threshold"]))
    for a_, b_ in zip(dets, dets2):
        assert [(d.cls_id, d.bbox, d.mask, d.conf) for d in a_.detections] == [(d.cls_id, d.bbox, d.mask, d.conf) for d in b_.detections]
    assert torch.equal(lazy_out.masks.materialize(), out.masks)


def test_bisenet_pair_blocks_run_as_pair_convs(ref_backend):
    """precision="fp32_tc": the stride-1 CatBottlenecks run in the pair format (concat buffer = channel slices of one pair buffer), the stride-2 blocks and the
    context path read the pairs through fp32-output convs - host bookkeeping on the CPU references, same results as the fp32 graph up to the pair rounding."""
    g = load_golden("bisenetformer_l_ade_b2_256x384")
    m = BisenetFormer(BisenetFormerConfig(), precision="fp32_tc")
    m.load_state_dict(seeded_state_dict(manifest_template("bisenetformer_l_ade"), 0), strict=True)
    eng = m.engine()
    H, W = (int(v) for v in g["sizes"][0])
    taken = [eng.trunk._pair_block_ok(blk, H // (8 << si), W // (8 << si)) for si, stage in enumerate(eng.trunk.blocks) for blk in stage]
    assert sum(taken) >= 6 and not any(t for t, blk in zip(taken, [b for st in eng.trunk.blocks for b in st]) if blk["stride"] == 2)
    imgs = synth_images(4, [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    ops._backend = calls = ConvCalls(ops._backend)
    out = m(x, taps=taps)
    pair_convs = [c for t, blk in zip(taken, [b for st in eng.trunk.blocks for b in st]) if t for c in blk["convs"]]
    paired = {id(w) for w in calls.w["conv2d_pair"]}
    assert all(id(c.w3) in paired for c in pair_convs)
    assert not any(c.w is w or c.w3 is w for c in pair_convs for w in calls.w["conv2d"])
    assert np.abs(taps["cp32"].permute(0, 3, 1, 2)[:, ::16].numpy() - g["cp32_tap"]).max() <= 1e-4 * np.abs(g["cp32_tap"]).max()
    assert np.abs(out.logits.numpy() - g["logits"]).max() <= 1e-3
    assert np.abs(out.masks[:, ::10, ::4, ::4].numpy() - g["masks_q10_s4"]).max() <= 1e-3
