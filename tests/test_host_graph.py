"""Host-side orchestration on a GPU-less machine: the fused NHWC graph of focoos_b200.fai_detr is run with the
per-operator CPU references (oracle/ops_ref.py) installed as the ops backend, and compared with the golden
fixtures produced by the unmodified reference.  This validates weight packing (BN fold, RepVGG re-param, fused
CSP / value_proj / offsets GEMMs), level ordering, concat slices and the processor — not the CUDA kernels."""
import numpy as np
import pytest
import torch

from focoos_b200 import FAIDetr, DETRConfig, DETRProcessor, ops
from focoos_b200.ports import DETRModelOutput
from oracle.gen_golden import synth_images
from oracle.ops_ref import RefBackend
from tests.parity_utils import ConvCalls, compare_queries, load_golden, manifest_template, seeded_sd


@pytest.fixture()
def ref_backend():
    ops._backend = RefBackend()
    yield
    ops._backend = None


def test_state_dict_keys_match_reference_manifest():
    m = FAIDetr(DETRConfig())
    own = {k: (tuple(v.shape), v.dtype) for k, v in m.state_dict().items()}
    ref = {k: (tuple(v.shape), v.dtype) for k, v in manifest_template().items()}
    assert own.keys() == ref.keys(), (sorted(set(own) ^ set(ref))[:10])
    assert own == ref


def test_no_cpu_fallback():
    m = FAIDetr(DETRConfig())
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 64, 64))


def test_fp32_tc_takes_only_the_default_algorithm():
    m = FAIDetr(DETRConfig(), precision="fp32_tc")
    m.algo = ops.ALGO_SIMT
    with pytest.raises(ValueError):
        m.engine()


def test_fused_graph_matches_golden(ref_backend):
    g = load_golden("detr_l_obj365_b2_640")
    m = FAIDetr(DETRConfig(), precision="fp32")
    m.load_state_dict(seeded_sd(0), strict=True)
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=torch.device("cpu"))
    taps = {}
    out = m(x, taps=taps)
    for t in ("res3", "res4", "res5"):
        v = taps[t].permute(0, 3, 1, 2)
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        assert np.abs(sl - g["tap_" + t]).max() <= 2e-4 * g["tapstat_" + t][2], t
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.numpy(), out.boxes.numpy(), taps["topk_ind"].numpy())
    assert ds < 2e-4 and db < 2e-4, (ds, db)
    dets = proc.postprocess(out, imgs, threshold=0.5)
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert sorted(x.cls_id for x in d.detections) == sorted(g["det_labels"][i, :n].tolist())
        assert sorted(tuple(x.bbox) for x in d.detections) == sorted(map(tuple, g["det_boxes"][i, :n].tolist()))


def test_processor_ragged_sizes(ref_backend):
    g = load_golden("detr_l_obj365_b3_ragged")
    sizes = [tuple(s) for s in g["image_sizes"].tolist()]
    imgs = synth_images(2, sizes)
    proc = DETRProcessor(DETRConfig(), image_size=640)
    x, _ = proc.preprocess(imgs, device=torch.device("cpu"))
    assert np.abs(x[:, :, 100:108, 200:208].numpy() - g["pre_image_patch"]).max() < 1e-3
    out = DETRModelOutput(boxes=torch.from_numpy(g["boxes"]), logits=torch.from_numpy(g["scores"]))
    dets = proc.postprocess(out, imgs, threshold=float(g["threshold"]))
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist() or sorted(x.cls_id for x in d.detections) == sorted(g["det_labels"][i, :n].tolist())
        assert sorted(tuple(x.bbox) for x in d.detections) == sorted(map(tuple, g["det_boxes"][i, :n].tolist()))


def test_fp32_tc_runs_only_pair_convs_and_matches_golden(ref_backend):
    """precision="fp32_tc" host orchestration (pair-format trunk, fused row glue of csrc/head_fused.cu in the AIFI / selection / decoder chains) through the CPU
    operator references: same golden bars as the fp32 graph, and the same selected queries, outputs and taps as the fp32 graph under the same references.
    Near-tied selection scores may come out in another order, so the queries are compared as sets and the per-query rows matched by encoder anchor."""
    g = load_golden("detr_l_obj365_b2_640")
    proc = DETRProcessor(DETRConfig(), image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=torch.device("cpu"))
    runs = {}
    for precision in ("fp32_tc", "fp32"):
        m = FAIDetr(DETRConfig(), precision=precision)
        m.load_state_dict(seeded_sd(0), strict=True)
        ops._backend = calls = ConvCalls(ops._backend)
        taps = {}
        runs[precision] = (m(x, taps=taps), taps)
        ops._backend = calls.be
        if precision == "fp32_tc":  # the pair flow runs every conv and linear through conv2d_pair: none goes to conv2d
            assert not calls.w["conv2d"] and calls.w["conv2d_pair"]
        else:
            assert calls.w["conv2d"] and not calls.w["conv2d_pair"]
    (a, ta), (b, tb) = runs["fp32_tc"], runs["fp32"]
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], a.logits.numpy(), a.boxes.numpy(), ta["topk_ind"].numpy())
    assert ds < 2e-4 and db < 2e-4, (ds, db)
    ka, kb = ta["topk_ind"], tb["topk_ind"]
    assert torch.equal(ka.sort(-1).values, kb.sort(-1).values)
    rows = torch.stack([kb[i].argsort()[ka[i].argsort().argsort()] for i in range(len(ka))])  # rows[i, j]: the fp32 row of the fp32_tc query j
    fp32_rows = lambda t: torch.stack([t[i][rows[i]] for i in range(len(t))])  # noqa: E731
    assert tuple(a.logits.shape) == tuple(b.logits.shape) and a.logits.is_contiguous()
    assert (a.logits - fp32_rows(b.logits)).abs().max() < 1e-5 and (a.boxes - fp32_rows(b.boxes)).abs().max() < 1e-5
    for k in ("aifi", "dec0_out", "dec5_out", "dec5_ref", "pred_logits"):
        want = tb[k] if k == "aifi" else fp32_rows(tb[k])
        assert (ta[k] - want).abs().max() <= 1e-4 * max(1.0, float(want.abs().max())), k
    dets = proc.postprocess(a, imgs, threshold=0.5)
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert sorted(tuple(x.bbox) for x in d.detections) == sorted(map(tuple, g["det_boxes"][i, :n].tolist()))
