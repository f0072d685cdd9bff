"""precision="fp32_tc" host orchestration of the three families on the CPU operator references: the split-precision tensor-core products - the engine's
convs and linears, and the per-query mask product of MaskFormer / BisenetFormer (per-image weights) - are reached only through conv2d_pair, and every
conv2d call is the fp32 CUDA-core conv on the fp32 storage weight (at 160x192 that includes MaskFormer's 1/32 encoder: under 64 tokens it stays on the
CUDA-core conv)."""
import pytest
import torch

from focoos_b200 import DETRConfig, FAIDetr, ops
from focoos_b200.bisenetformer import BisenetFormer, BisenetFormerConfig
from focoos_b200.fai_mf import FAIMaskFormer, MaskFormerConfig
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import ConvCalls, manifest_template

FAMILIES = {"fai_detr": (FAIDetr, DETRConfig, "fai_detr_l_obj365"),
            "fai_mf": (FAIMaskFormer, MaskFormerConfig, "fai_mf_l_coco_ins"),
            "bisenetformer": (BisenetFormer, BisenetFormerConfig, "bisenetformer_l_ade")}


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


@pytest.mark.parametrize("family", list(FAMILIES))
def test_fp32_tc_reaches_split_products_only_through_conv2d_pair(ref_backend, family):
    cls, cfg, manifest = FAMILIES[family]
    m = cls(cfg(), precision="fp32_tc")
    m.load_state_dict(seeded_state_dict(manifest_template(manifest), 0), strict=True)
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in synth_images(3, [(160, 192)])])
    ops._backend = calls = ConvCalls(ops._backend)
    m(x)
    assert calls.w["conv2d_pair"]
    assert any(w.dim() == 5 for w in calls.w["conv2d_pair"]) == (family != "fai_detr"), "the mask product runs as conv2d_pair with per-image weights"
    assert all(w.dtype == torch.float32 for w in calls.w["conv2d"]), sorted({str(w.dtype) for w in calls.w["conv2d"]})
