"""fai-detr-m-coco (the DETR family on the STDC-2 trunk, no AIFI layer, 3 decoder layers) on a GPU-less machine: configuration, module tree, registry, export
meta and training guard, and the fused NHWC graph run with the per-operator CPU references (oracle/ops_ref.py) against the fixtures of the unmodified
reference (oracle/gen_golden_detr_m.py)."""
import json
import os

import numpy as np
import pytest
import torch

from focoos_b200 import FAIDetr, DETRConfig, DETRProcessor, ops
from focoos_b200.export import _rebuild, make_meta
from focoos_b200.trunks import STDC
from focoos_b200.model_manager import _REGISTRY, ModelManager
from focoos_b200.ports import ResnetConfig, STDCConfig
from focoos_b200.trainer import TrainerArgs, run_train_entry
from oracle.gen_golden import state_dict_digest, synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import GOLDEN, ConvCalls, compare_queries, load_golden, manifest_template, seeded_sd

NAME, MANIFEST, TAG = "fai-detr-m-coco", "fai_detr_m_coco", "detr_m_coco_b2_640"


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


def _config():
    return DETRConfig.from_dict(_REGISTRY[NAME]["config"])


def _model(precision):
    m = FAIDetr(_config(), precision=precision)
    m.load_state_dict(seeded_sd(0, MANIFEST), strict=True)
    return m


def _check_keep_sets(g, dets):
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert sorted((x.cls_id, tuple(x.bbox)) for x in d.detections) == sorted(zip(g["det_labels"][i, :n].tolist(), map(tuple, g["det_boxes"][i, :n].tolist())))


def _check_backbone_taps(g, taps):
    for t in ("res3", "res4", "res5"):
        v = taps[t].permute(0, 3, 1, 2)
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        assert np.abs(sl - g["tap_" + t]).max() <= 2e-4 * g["tapstat_" + t][2], t


def test_state_dict_matches_reference_manifest():
    m = FAIDetr(_config())
    own = {k: (tuple(v.shape), v.dtype) for k, v in m.state_dict().items()}
    ref = {k: (tuple(v.shape), v.dtype) for k, v in manifest_template(MANIFEST).items()}
    assert len(ref) == 679
    assert own.keys() == ref.keys(), sorted(set(own) ^ set(ref))[:10]
    assert own == ref
    assert not any(k.startswith("pixel_decoder.encoder.") for k in own)


def test_config_picks_the_backbone_from_model_type():
    cfg = _config()
    assert isinstance(cfg.backbone_config, STDCConfig) and cfg.backbone_config.layers == [4, 5, 3]
    assert cfg.pixel_decoder_num_encoder_layers == 0 and cfg.transformer_predictor_dec_layers == 3
    assert isinstance(DETRConfig.from_dict({"backbone_config": {"model_type": "resnet", "depth": 50}}).backbone_config, ResnetConfig)
    assert isinstance(DETRConfig.from_dict({}).backbone_config, ResnetConfig)
    with pytest.raises(ValueError, match="model_type"):
        DETRConfig.from_dict({"backbone_config": {"model_type": "mobilenet"}})
    with pytest.raises(ValueError, match="pixel_decoder_num_encoder_layers"):
        DETRConfig.from_dict({"pixel_decoder_num_encoder_layers": 2})
    with pytest.raises(ValueError, match="pixel_decoder_num_encoder_layers"):
        DETRConfig(pixel_decoder_num_encoder_layers=2)


def test_model_manager_serves_the_model():
    fm = ModelManager.get(NAME)
    assert type(fm.model) is FAIDetr and isinstance(fm.model.pixel_decoder.backbone, STDC)
    assert type(fm.processor) is DETRProcessor and fm.processor.image_size == 640
    assert fm.model.num_classes == 80


def test_fused_graph_matches_golden(ref_backend):
    g = load_golden(TAG)
    with open(os.path.join(GOLDEN, "golden_meta_detr_m.json")) as f:
        assert state_dict_digest(seeded_sd(0, MANIFEST)) == json.load(f)["weights_sha256"]
    m = _model("fp32")
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=torch.device("cpu"))
    taps = {}
    out = m(x, taps=taps)
    assert "aifi" not in taps
    _check_backbone_taps(g, taps)
    for t in ("fpn0", "fpn1", "pan0", "pan1"):
        v = taps[t].permute(0, 3, 1, 2)
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        assert np.abs(sl - g["tap_" + t]).max() <= 2e-4 * g["tapstat_" + t][2], t
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.numpy(), out.boxes.numpy(), taps["topk_ind"].numpy())
    assert ds < 2e-4 and db < 2e-4, (ds, db)
    _check_keep_sets(g, proc.postprocess(out, imgs, threshold=0.5))


def test_fp32_tc_runs_only_pair_convs_and_matches_golden(ref_backend):
    g = load_golden(TAG)
    m = _model("fp32_tc")
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=torch.device("cpu"))
    ops._backend = calls = ConvCalls(ops._backend)
    taps = {}
    out = m(x, taps=taps)
    ops._backend = calls.be
    assert not calls.w["conv2d"] and calls.w["conv2d_pair"]
    eng = m.engine()
    assert any(eng.trunk._pair_block_ok(blk, 640 // (8 << si), 640 // (8 << si)) for si, stage in enumerate(eng.trunk.blocks) for blk in stage)
    _check_backbone_taps(g, taps)
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.numpy(), out.boxes.numpy(), taps["topk_ind"].numpy())
    assert ds < 2e-4 and db < 2e-4, (ds, db)
    _check_keep_sets(g, proc.postprocess(out, imgs, threshold=0.5))


def test_export_meta_rebuilds_the_stdc_trunk():
    m = FAIDetr(_config(), precision="fp32_tc")
    sd = m.state_dict()
    r = _rebuild(make_meta(m), list(sd.values()))
    assert isinstance(r.config.backbone_config, STDCConfig) and isinstance(r.pixel_decoder.backbone, STDC)
    assert r.precision == "fp32_tc" and r.config == m.config
    assert all(torch.equal(a, b) for a, b in zip(r.state_dict().values(), sd.values()))


def test_training_entry_raises_for_the_stdc_trunk(tmp_path):
    fm = ModelManager.get(NAME)
    with pytest.raises(NotImplementedError, match="backward kernels"):
        run_train_entry(fm, TrainerArgs(run_name="m", output_dir=str(tmp_path), num_gpus=1), data_train=None)
    assert not any(tmp_path.iterdir())
    with pytest.raises(NotImplementedError, match="backward kernels"):
        fm.model.train_graph()
