"""-m gpu: fai-detr-m-coco (STDC-2 trunk, hybrid encoder at width 128 without an AIFI layer, 3 decoder layers, 80 classes) end to end on the CUDA path,
against the fixtures of the unmodified reference (oracle/gen_golden_detr_m.py).  Bars as for fai-detr-l (tests/test_gpu_e2e.py): fp32 and fp32_tc with
identical query sets, scores and boxes within 1e-3 and identical keep-sets; fp16 measured with looser asserts."""
import numpy as np
import pytest
import torch

from focoos_b200 import DETRConfig, DETRProcessor, FAIDetr, FocoosModel, ModelInfo, ops
from focoos_b200.model_manager import _REGISTRY
from oracle.gen_golden import synth_images
from tests.parity_utils import compare_queries, load_golden, seeded_sd, update_report

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

NAME, TAG = "fai-detr-m-coco", "detr_m_coco_b2_640"


@pytest.fixture(scope="module")
def sd():
    return seeded_sd(0, "fai_detr_m_coco")


def _model(sd, precision, algo=ops.ALGO_AUTO):
    m = FAIDetr(DETRConfig.from_dict(_REGISTRY[NAME]["config"]), precision=precision)
    m.load_state_dict(sd, strict=True)
    m.cuda()
    m.algo = algo
    return m


def _run_golden(sd, precision, algo=ops.ALGO_AUTO, trace=False):
    m = _model(sd, precision, algo)
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=m.device)
    taps = {}
    tr = ops.enable_trace() if trace else None
    try:
        out = m(x, taps=taps)
        torch.cuda.synchronize()
    finally:
        if trace:
            ops.enable_trace(False)
    return m, proc, imgs, out, taps, tr


def _backbone_rel_err(g, taps):
    rel = {}
    for t in ("res3", "res4", "res5"):
        v = taps[t].permute(0, 3, 1, 2).float().cpu()
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        rel[t] = float(np.abs(sl - g["tap_" + t]).max() / g["tapstat_" + t][2])
    return rel


def _overlap(key_a, key_b):
    return [len(set(a.tolist()) & set(b.tolist())) for a, b in zip(key_a, key_b)]


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
def test_fp32_modes_match_reference_golden(sd, precision):
    g = load_golden(TAG)
    m, proc, imgs, out, taps, trace = _run_golden(sd, precision, trace=precision == "fp32_tc")
    if precision == "fp32_tc":
        symbols = [e[0] for e in trace]
        assert "fb200_conv2d_pair" in symbols and "fb200_conv2d" not in symbols, "every conv / linear of the fp32_tc flow runs as conv2d_pair"
    rel = _backbone_rel_err(g, taps)
    assert all(v <= 2e-4 for v in rel.values()), rel
    keys = taps["topk_ind"].cpu().numpy()
    assert _overlap(g["enc_topk_ind"], keys) == [300, 300], "encoder query SETS must be identical"
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.cpu().numpy(), out.boxes.cpu().numpy(), keys)
    update_report("parity_report.json", {f"detr_m_{precision}_vs_reference_golden": {"scores_max_abs": ds, "boxes_max_abs": db}})
    assert ds < 1e-3 and db < 1e-3, (ds, db)
    for i, d in enumerate(proc.postprocess(out, imgs, threshold=0.5)):
        n = int(g["det_count"][i])
        assert len(d) == n, "keep-set size"
        assert sorted((x.cls_id, tuple(x.bbox)) for x in d.detections) == sorted(zip(g["det_labels"][i, :n].tolist(), map(tuple, g["det_boxes"][i, :n].tolist())))


@pytest.mark.parametrize("algo,name", [(ops.ALGO_SIMT, "fp16_simt"), (ops.ALGO_AUTO, "fp16_auto")])
def test_fp16_vs_reference_golden(sd, algo, name):
    g = load_golden(TAG)
    _, _, _, out, taps, _ = _run_golden(sd, "fp16", algo)
    rel = _backbone_rel_err(g, taps)
    overlap = _overlap(g["enc_topk_ind"], taps["topk_ind"].cpu().numpy())
    update_report("parity_report.json", {f"detr_m_{name}": {"backbone_rel_err": rel, "enc_query_overlap_of_300": overlap}})
    assert all(v < 2e-2 for v in rel.values()), rel
    assert min(overlap) >= 240, overlap
    assert torch.isfinite(out.logits).all() and torch.isfinite(out.boxes).all()


@pytest.mark.parametrize("precision", ["fp16", "fp32_tc"])
def test_batch_invariance_at_bs32(sd, precision):
    """per-image results do not depend on the batch they were computed in (bit-exact) at the benchmark's batch size"""
    m = _model(sd, precision)
    x = torch.from_numpy(np.stack(synth_images(21, [(640, 640)] * 32))).cuda()
    out32 = m(x)
    out4 = m(x[4:8].contiguous())
    assert torch.equal(out32.logits[4:8], out4.logits) and torch.equal(out32.boxes[4:8], out4.boxes)
    assert tuple(out32.logits.shape) == (32, 300, 80)


def test_focoos_model_cuda_graph_path_equals_eager(sd):
    fm = FocoosModel(_model(sd, "fp32_tc"), ModelInfo(name=NAME, im_size=640))
    batches = [np.stack(synth_images(s, [(640, 640)] * 2)) for s in (1, 2)]
    fm.cuda_graphs = False
    ref = [fm(torch.from_numpy(b), threshold=0.5, batched=True) for b in batches]
    fm.cuda_graphs = True
    for rep in range(3):  # call 1 eager, call 2 captures, call 3+ replay
        for b, r in zip(batches, ref):
            got = fm(torch.from_numpy(b), threshold=0.5, batched=True)
            for g, e in zip(got, r):
                assert [(d.cls_id, d.bbox, d.conf) for d in g.detections] == [(d.cls_id, d.bbox, d.conf) for d in e.detections], rep
    assert len(fm._graphs) == 1


def test_pipelined_inference_equals_the_synchronous_call(sd):
    fm = FocoosModel(_model(sd, "fp16"), ModelInfo(name=NAME, im_size=640))
    batches = [torch.from_numpy(np.stack(synth_images(s, [(640, 640)] * 2))).pin_memory() for s in (1, 2, 3, 4)]
    ref = [fm(b, threshold=0.5, batched=True) for b in batches]
    key = lambda dets: [[(d.cls_id, tuple(d.bbox), d.conf) for d in x.detections] for x in dets]  # noqa: E731
    assert [key(g) for g in fm.stream(batches, threshold=0.5)] == [key(r) for r in ref]
    assert key(fm.infer_async(batches[1], threshold=0.5).result()) == key(ref[1])


def test_export_roundtrip_on_gpu(sd, tmp_path):
    """the TorchScript export rebuilds the STDC trunk from its meta and reproduces the eager fp32_tc tensors bit for bit"""
    fm = FocoosModel(_model(sd, "fp32_tc"), ModelInfo(name=NAME, im_size=640))
    fm.export(out_dir=str(tmp_path), image_size=640)
    x = 128 * torch.randn(2, 3, 640, 640, device="cuda")
    eager = fm.model(x)
    boxes, logits = torch.jit.load(str(tmp_path / "model.pt"))(x)
    assert torch.equal(boxes, eager.boxes) and torch.equal(logits, eager.logits)
