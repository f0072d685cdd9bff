"""fai-mf-m-coco-ins and fai-mf-s-coco-ins (128-wide TransformerFPN, 8 encoder heads of 16 channels) on a GPU-less machine: registry config, module tree
against the reference manifest, the fp32 / fp32_tc host graphs on the CPU operator references against golden fixtures produced by the unmodified reference
(oracle/gen_golden_mf_128.py), and the export meta rebuilding the model."""
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from focoos_b200 import FAIMaskFormer, ModelManager, ops
from focoos_b200.export import _rebuild, make_meta
from focoos_b200.fai_mf import MaskFormerConfig
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import state_dict_digest, synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import GOLDEN, load_golden, manifest_template

MODELS = {"fai-mf-m-coco-ins": ("mf_m_coco_ins", 101), "fai-mf-s-coco-ins": ("mf_s_coco_ins", 50)}


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


def _meta():
    with open(os.path.join(GOLDEN, "golden_meta_mf_128.json")) as f:
        return json.load(f)


def _model(name, precision):
    m = ModelManager.get(name, precision=precision).model
    sd = seeded_state_dict(manifest_template("fai_" + MODELS[name][0]), 0)
    m.load_state_dict(sd, strict=True)
    return m, sd


@pytest.mark.parametrize("name", list(MODELS))
def test_config_from_registry(name):
    fm = ModelManager.get(name)
    c = fm.model.config
    assert isinstance(fm.model, FAIMaskFormer) and fm.model_info.im_size == 1024 and c.resolution == 1024
    assert c.backbone_config.depth == MODELS[name][1]
    assert (c.pixel_decoder_feat_dim, c.pixel_decoder_out_dim, c.pixel_decoder_transformer_layers, c.pixel_decoder_transformer_nheads) == (128, 128, 3, 8)
    assert (c.transformer_predictor_hidden_dim, c.transformer_predictor_out_dim, c.transformer_predictor_dec_layers, c.transformer_predictor_dim_feedforward) == (256, 128, 6, 1024)
    assert (c.head_out_dim, c.postprocessing_type, c.num_classes, c.num_queries) == (128, "instance", 80, 100)


@pytest.mark.parametrize("name", list(MODELS))
def test_module_tree_matches_reference_manifest(name):
    m = ModelManager.get(name).model
    own = {k: (tuple(v.shape), v.dtype) for k, v in m.state_dict().items()}
    ref = {k: (tuple(v.shape), v.dtype) for k, v in manifest_template("fai_" + MODELS[name][0]).items()}
    assert own.keys() == ref.keys(), sorted(set(own) ^ set(ref))[:10]
    assert own == ref


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
@pytest.mark.parametrize("fixture", ["mf_m_coco_ins_b2_320x416", "mf_s_coco_ins_b2_320x416", "mf_s_coco_ins_b2_357x483"])
def test_host_graph_matches_golden(ref_backend, fixture, precision):
    meta = _meta()[fixture]
    g = load_golden(fixture)
    m, sd = _model(meta["model"], precision)
    assert state_dict_digest(sd) == meta["weights_sha256"]
    eng = m.engine()
    assert (eng.pd_d, eng.pd_nhead, eng.d, eng.nhead) == (128, 8, 256, 8)
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    out = m(x, taps=taps)
    assert tuple(out.masks.shape[-2:]) == tuple(g["sizes"][0])
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2).float()  # NHWC -> [B,Q,h,w]
    ref_pm, pm = g["pred_masks_q10_s2"], pm[:, ::10, ::2, ::2]
    # the bars of the fai-mf-l-coco-ins host-graph tests: pre-sigmoid mask logits relative to their scale, probabilities absolute
    e_logit = float(np.abs(pm.numpy() - ref_pm).max())
    e_cls = float(np.abs(out.logits.numpy() - g["logits"]).max())
    e_mask = float(np.abs(out.masks[:, ::10, ::4, ::4].numpy() - g["masks_q10_s4"]).max())
    fp32 = precision == "fp32"
    assert e_logit <= (1e-4 if fp32 else 1e-3) * scale and e_cls <= 1e-3 and e_mask <= (1e-3 if fp32 else 2e-3), (e_logit, e_cls, e_mask)
    if "enc_memory_tap" in g:  # the 128-wide encoder output, NHWC here, [B,C,h,w] in the reference
        enc = taps["enc_memory"].permute(0, 3, 1, 2)[:, ::32].numpy()
        assert np.abs(enc - g["enc_memory_tap"]).max() <= 1e-3 * max(1.0, float(np.abs(g["enc_memory_tap"]).max()))
    dets = MaskFormerProcessor(m.config).postprocess(out, imgs, threshold=float(g["threshold"]))
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        if n:
            assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() < 1e-3
            assert np.abs(np.array([x.bbox for x in d.detections]) - g["det_boxes"][i, :n]).max() <= (0 if fp32 else 3)


@pytest.mark.parametrize("name", list(MODELS))
def test_export_meta_rebuilds_the_model(ref_backend, name):
    """the TorchScript file carries asdict(config) in its meta; rebuilding from it gives the same 128-wide model and the same outputs"""
    m, sd = _model(name, "fp32")
    meta = make_meta(m)
    assert json.loads(meta)["family"] == "fai_mf"
    r = _rebuild(meta, [t for _, t in m.state_dict().items()])
    assert type(r) is FAIMaskFormer and asdict(r.config) == asdict(m.config) and r.precision == "fp32"
    assert r.config == MaskFormerConfig.from_dict(json.loads(meta)["config"])
    x = synth_images(3, [(64, 96)])
    x = torch.from_numpy(x[0]).permute(2, 0, 1).float()[None]
    a, b = m(x), r(x)
    assert torch.equal(a.logits, b.logits) and torch.equal(a.masks, b.masks)
