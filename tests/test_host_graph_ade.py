"""The ADE20K semantic segmenters (fai-mf-l-ade, fai-mf-m-ade, bisenetformer-m-ade, bisenetformer-s-ade) on a GPU-less machine: registry entries, config
parsing, module trees against the reference manifests, the fp32 / fp32_tc host graphs on the CPU operator references against golden fixtures produced by
the unmodified reference (oracle/gen_golden_ade.py), the lazy semantic path, the pair flow of the encoder-less pixel decoder, and the export meta."""
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from focoos_b200 import FAIMaskFormer, ModelManager, ops
from focoos_b200.bisenetformer import BisenetFormer
from focoos_b200.export import _rebuild, make_meta
from focoos_b200.trunks import STDC, ResNet
from focoos_b200.fai_mf import MaskFormerConfig
from focoos_b200.ports import ResnetConfig, STDCConfig
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import state_dict_digest, synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import GOLDEN, ConvCalls, load_golden, manifest_template

# name -> (model class, trunk class, manifest, state_dict key count of the reference)
MODELS = {
    "fai-mf-l-ade": (FAIMaskFormer, ResNet, "fai_mf_l_ade", 807),
    "fai-mf-m-ade": (FAIMaskFormer, STDC, "fai_mf_m_ade", 435),
    "bisenetformer-m-ade": (BisenetFormer, STDC, "bisenetformer_m_ade", 469),
    "bisenetformer-s-ade": (BisenetFormer, STDC, "bisenetformer_s_ade", 361),
}
FIXTURES = ["mf_l_ade_b2_320x416", "mf_m_ade_b2_320x416", "mf_m_ade_b2_357x483", "bisenetformer_m_ade_b2_256x384", "bisenetformer_m_ade_b2_357x483",
            "bisenetformer_s_ade_b2_256x384"]

# The masked decoder turns tiny differences into flipped attention-mask bits (logit < 0), which the seeded, peaky weights amplify (DESIGN.md §2):
#  * fai-mf-l-ade (mask logits up to |130|) is chaotic on its golden: the fp32 flow itself, fed the same images times (1 + 1e-6 noise), moves the class
#    probabilities by 0.07 and the mask probabilities by 0.23 while its mask features move by 4e-6.  fp32 follows the reference's operation order closely
#    enough to meet the bars; fp32_tc (mask features 5e-6 off) lands inside that spread.
#  * fai-mf-m-ade at 357x483 in fp32: one flipped bit puts the class probabilities 2.9e-3 off; mask logits, mask probabilities and detections meet the bars.
CHAOTIC = {("mf_l_ade_b2_320x416", "fp32_tc")}
CLS_BAR = {("mf_m_ade_b2_357x483", "fp32"): 4e-3}


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


def _meta():
    with open(os.path.join(GOLDEN, "golden_meta_ade.json")) as f:
        return json.load(f)


def _model(name, precision):
    m = ModelManager.get(name, precision=precision).model
    sd = seeded_state_dict(manifest_template(MODELS[name][2]), 0)
    m.load_state_dict(sd, strict=True)
    return m, sd


def _masks_sample(g, masks):
    """the final probabilities the fixture holds: every 10th query (masks_q10_s4) or, in the odd-size files, every 20th (masks_q20_s4), at every 4th pixel"""
    key = "masks_q10_s4" if "masks_q10_s4" in g else "masks_q20_s4"
    q = 10 if key == "masks_q10_s4" else 20
    return masks[:, ::q, ::4, ::4], g[key]


@pytest.mark.parametrize("name", list(MODELS))
def test_module_tree_matches_reference_manifest(name):
    m = ModelManager.get(name).model
    own = {k: (tuple(v.shape), v.dtype) for k, v in m.state_dict().items()}
    ref = {k: (tuple(v.shape), v.dtype) for k, v in manifest_template(MODELS[name][2]).items()}
    assert len(ref) == MODELS[name][3]
    assert own.keys() == ref.keys(), sorted(set(own) ^ set(ref))[:10]
    assert own == ref


@pytest.mark.parametrize("name", list(MODELS))
def test_registry_builds_class_trunk_and_processor(name):
    fm = ModelManager.get(name)
    cls, trunk, _, _ = MODELS[name]
    m, c = fm.model, fm.model.config
    assert type(m) is cls and type(m.pixel_decoder.backbone) is trunk
    assert isinstance(fm.processor, MaskFormerProcessor) and fm.processor.predict_all_pixels and not fm.processor.use_mask_score
    assert fm.model_info.im_size == 640 and fm.model_info.model_family == ("fai_mf" if cls is FAIMaskFormer else "bisenetformer")
    assert (c.num_classes, c.num_queries, c.postprocessing_type, c.predict_all_pixels, c.use_mask_score) == (150, 100, "semantic", True, False)
    if cls is FAIMaskFormer:
        pd = m.pixel_decoder
        assert c.pixel_decoder_transformer_layers == 0 and not hasattr(pd, "input_proj") and not hasattr(pd, "transformer")
        assert pd.layer_4.in_channels == pd.backbone.out_channels[3]  # 2048 (R101-vd), 1024 (STDC-2)
        assert c.transformer_predictor_dec_layers == (6 if name == "fai-mf-l-ade" else 3)
    if name == "bisenetformer-m-ade":
        assert (c.pixel_decoder_feat_dim, c.pixel_decoder_out_dim, c.transformer_predictor_dec_layers, c.transformer_predictor_dim_feedforward) == (96, 96, 4, 512)
    if name == "bisenetformer-s-ade":
        assert c.backbone_config.layers == [2, 2, 2]


def test_maskformer_config_chooses_the_trunk():
    stdc = MaskFormerConfig.from_dict({"backbone_config": {"model_type": "stdc", "base": 64, "layers": [4, 5, 3], "unknown_field": 1}})
    assert isinstance(stdc.backbone_config, STDCConfig) and stdc.backbone_config.layers == [4, 5, 3]
    assert isinstance(MaskFormerConfig.from_dict({"backbone_config": {"model_type": "resnet", "depth": 50}}).backbone_config, ResnetConfig)
    assert isinstance(MaskFormerConfig.from_dict({"backbone_config": {"depth": 50}}).backbone_config, ResnetConfig)  # no model_type: ResNet, as before
    with pytest.raises(ValueError, match="model_type for MaskFormerConfig: 'mobilenet'"):
        MaskFormerConfig.from_dict({"backbone_config": {"model_type": "mobilenet"}})


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
@pytest.mark.parametrize("fixture", FIXTURES)
def test_host_graph_matches_golden(ref_backend, fixture, precision):
    meta = _meta()[fixture]
    g = load_golden(fixture)
    m, sd = _model(meta["model"], precision)
    assert state_dict_digest(sd) == meta["weights_sha256"]
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    taps = {}
    out = m(x, taps=taps)
    assert tuple(out.masks.shape[-2:]) == tuple(g["sizes"][0])
    assert "enc_memory" not in taps
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2).float()  # NHWC -> [B,Q,h,w]
    e_logit = float(np.abs(pm[:, ::10, ::2, ::2].numpy() - g["pred_masks_q10_s2"]).max())
    e_cls = float(np.abs(out.logits.numpy() - g["logits"]).max())
    got, ref = _masks_sample(g, out.masks)
    e_mask = float(np.abs(got.numpy() - ref).max())
    fp32 = precision == "fp32"
    if "mask_features_tap" in g:
        mf = taps["mask_features"].permute(0, 3, 1, 2)[:, ::16, ::4, ::4].float().numpy()
        assert np.abs(mf - g["mask_features_tap"]).max() <= 1e-4 * np.abs(g["mask_features_tap"]).max()
    if (fixture, precision) in CHAOTIC:
        # see CHAOTIC: the pixel decoder (the tap above) is held to 1e-4 of its scale, the decoder outputs to the spread a 1e-6 input perturbation causes
        assert e_logit <= 0.05 * scale and e_cls <= 0.1 and e_mask <= 0.3, (e_logit, e_cls, e_mask)
        return
    # the bars of the fai-mf / bisenetformer host-graph tests: pre-sigmoid mask logits relative to their scale, probabilities absolute
    assert e_logit <= (1e-4 if fp32 else 1e-3) * scale and e_cls <= CLS_BAR.get((fixture, precision), 1e-3) and e_mask <= (1e-3 if fp32 else 2e-3), (e_logit, e_cls, e_mask)
    dets = MaskFormerProcessor(m.config).postprocess(out, imgs, threshold=float(g["threshold"]))
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        if n:
            assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() < 1e-3
            assert np.abs(np.array([x.bbox for x in d.detections]) - g["det_boxes"][i, :n]).max() <= (0 if fp32 else 3)


@pytest.mark.parametrize("fixture", ["mf_m_ade_b2_320x416", "bisenetformer_m_ade_b2_256x384"])
def test_lazy_semantic_path_equals_materialised(ref_backend, fixture):
    """the lazy path (what FocoosModel.__call__ uses): semantic argmax straight from the low-resolution logits - the same detections"""
    meta = _meta()[fixture]
    g = load_golden(fixture)
    m, _ = _model(meta["model"], "fp32")
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    out = m(x)
    m.lazy_masks = True
    lazy_out = m(x)
    m.lazy_masks = False
    assert hasattr(lazy_out.masks, "materialize") and tuple(lazy_out.masks.shape) == tuple(out.masks.shape)
    proc = MaskFormerProcessor(m.config)
    dets, dets2 = proc.postprocess(out, imgs, threshold=0.5), proc.postprocess(lazy_out, imgs, threshold=0.5)
    assert sum(len(d) for d in dets) > 0
    for a_, b_ in zip(dets, dets2):
        assert [(d.cls_id, d.bbox, d.mask, d.conf) for d in a_.detections] == [(d.cls_id, d.bbox, d.mask, d.conf) for d in b_.detections]
    assert torch.equal(lazy_out.masks.materialize(), out.masks)


def test_mf_l_ade_pair_flow_runs_trunk_and_layer_4_as_pair_convs(ref_backend):
    """fp32_tc, fai-mf-l-ade: without an encoder, res5 (a Pair) goes straight into layer_4 - it and every trunk conv run as conv2d_pair on their weight triples,
    none on the fp32 conv"""
    m, _ = _model("fai-mf-l-ade", "fp32_tc")
    eng = m.engine()
    assert eng.pd_in is None and eng.enc == [] and eng.enc_norm is None
    layers = [eng.trunk.stem2, eng.trunk.stem3, *[blk[k] for st in eng.trunk.stages for blk in st for k in ("a", "b", "c", "short") if blk[k] is not None], eng.layer[4]]
    assert all(any(layer is p for p in eng._pair_layers()) for layer in layers)
    ops._backend = calls = ConvCalls(ops._backend)
    m(torch.from_numpy(synth_images(5, [(96, 128)])[0]).permute(2, 0, 1).float()[None])
    paired = {id(w) for w in calls.w["conv2d_pair"]}
    assert all(id(layer.w3) in paired for layer in layers)
    assert not any(layer.w is w or layer.w3 is w for layer in layers for w in calls.w["conv2d"])


def test_mf_m_ade_pair_layers_name_the_stdc_trunk():
    """fp32_tc, fai-mf-m-ade: the pair-flow layer set names what the STDC packing made (second stem, CatBottleneck convs) and layer_4, and each has its
    weight triple"""
    m, _ = _model("fai-mf-m-ade", "fp32_tc")
    eng = m.engine()
    pl = eng._pair_layers()
    stdc = [eng.trunk.stem2, *[c for st in eng.trunk.blocks for blk in st for c in blk["convs"]], eng.layer[4]]
    assert all(any(layer is p for p in pl) for layer in stdc) and all(layer.w3 is not None for layer in pl)


def test_export_meta_rebuilds_the_stdc_maskformer(ref_backend):
    """the TorchScript file carries asdict(config) in its meta; rebuilding from it gives fai-mf-m-ade with its STDC trunk and the same outputs"""
    m, sd = _model("fai-mf-m-ade", "fp32")
    meta = make_meta(m)
    assert json.loads(meta)["family"] == "fai_mf"
    r = _rebuild(meta, [t for _, t in m.state_dict().items()])
    assert type(r) is FAIMaskFormer and type(r.pixel_decoder.backbone) is STDC and isinstance(r.config.backbone_config, STDCConfig)
    assert asdict(r.config) == asdict(m.config) and r.precision == "fp32"
    x = torch.from_numpy(synth_images(3, [(64, 96)])[0]).permute(2, 0, 1).float()[None]
    a, b = m(x), r(x)
    assert torch.equal(a.logits, b.logits) and torch.equal(a.masks, b.masks)
