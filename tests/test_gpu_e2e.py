"""-m gpu: end-to-end parity of the CUDA path (through FAIDetr / DETRProcessor / the C ABI) against
(a) the golden fixtures produced by the unmodified reference and (b) the CPU oracle on fresh seeded inputs.

Bars (BASELINE.json north_star): class indices and top-k∧threshold keep-sets bit-exact, box coords within 1e-3 abs.
fp32 mode is held to those bars.  fp16 mode (the reference's own CUDA numerics class: it runs under fp16 autocast,
focoos_model.py:604-609) is measured and reported in parity_report.json (tests/parity_utils.update_report) with looser asserts."""

import numpy as np
import pytest
import torch

from focoos_b200 import DETRConfig, DETRProcessor, FAIDetr, ops
from oracle import detr_oracle as O
from oracle.gen_golden import synth_images
from tests.parity_utils import compare_queries, load_golden, seeded_sd, update_report

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _report(key, val):
    update_report("parity_report.json", {key: val})


@pytest.fixture(scope="module")
def sd():
    return seeded_sd(0)


def _model(sd, precision, algo=ops.ALGO_AUTO):
    m = FAIDetr(DETRConfig(), precision=precision)
    m.load_state_dict(sd, strict=True)
    m.cuda()
    m.algo = algo
    return m


def _set_stats(key_a, key_b):
    return [len(set(a.tolist()) & set(b.tolist())) for a, b in zip(key_a, key_b)]


def _common_err(g_scores, g_boxes, g_keys, scores, boxes, keys):
    """max abs diff over the queries both sides selected."""
    ds = db = 0.0
    for i in range(len(g_keys)):
        pos = {int(k): j for j, k in enumerate(keys[i].tolist())}
        rows = [(j, pos[int(k)]) for j, k in enumerate(g_keys[i].tolist()) if int(k) in pos]
        if not rows:
            continue
        a, b = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
        ds = max(ds, float(np.abs(g_scores[i][a] - scores[i][b]).max()))
        db = max(db, float(np.abs(g_boxes[i][a] - boxes[i][b]).max()))
    return ds, db


def test_fp32_matches_reference_golden(sd):
    g = load_golden("detr_l_obj365_b2_640")
    m = _model(sd, "fp32")
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=m.device)
    taps = {}
    out = m(x, taps=taps)
    torch.cuda.synchronize()
    for t in ("res3", "res4", "res5"):
        v = taps[t].permute(0, 3, 1, 2).float().cpu()
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        assert np.abs(sl - g["tap_" + t]).max() <= 2e-4 * g["tapstat_" + t][2], t
    keys = taps["topk_ind"].cpu().numpy()
    assert _set_stats(g["enc_topk_ind"], keys) == [300, 300], "encoder query SETS must be identical"
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.cpu().numpy(), out.boxes.cpu().numpy(), keys)
    _report("fp32_vs_reference_golden", {"scores_max_abs": ds, "boxes_max_abs": db})
    assert ds < 1e-3 and db < 1e-3, (ds, db)
    dets = proc.postprocess(out, imgs, threshold=0.5)
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n, "keep-set size"
        assert sorted(x.cls_id for x in d.detections) == sorted(g["det_labels"][i, :n].tolist()), "class indices"
        assert sorted(tuple(x.bbox) for x in d.detections) == sorted(map(tuple, g["det_boxes"][i, :n].tolist())), "keep-set boxes"
        confs = [x.conf for x in d.detections]
        assert confs == sorted(confs, reverse=True)


def test_fp32_ragged_golden(sd):
    g = load_golden("detr_l_obj365_b3_ragged")
    sizes = [tuple(s) for s in g["image_sizes"].tolist()]
    imgs = synth_images(2, sizes)
    m = _model(sd, "fp32")
    proc = DETRProcessor(m.config, image_size=640)
    x, _ = proc.preprocess(imgs, device=m.device)
    assert np.abs(x[:, :, 100:108, 200:208].cpu().numpy() - g["pre_image_patch"]).max() < 1e-3
    taps = {}
    out = m(x, taps=taps)
    keys = taps["topk_ind"].cpu().numpy()
    assert _set_stats(g["enc_topk_ind"], keys) == [300] * 3
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.cpu().numpy(), out.boxes.cpu().numpy(), keys)
    assert ds < 1e-3 and db < 1e-3, (ds, db)
    dets = proc.postprocess(out, imgs, threshold=float(g["threshold"]))
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert sorted(x.cls_id for x in d.detections) == sorted(g["det_labels"][i, :n].tolist())
        gb = np.array(sorted(map(tuple, g["det_boxes"][i, :n].tolist())))
        ob = np.array(sorted(tuple(x.bbox) for x in d.detections))
        assert np.abs(gb - ob).max() <= 1


def test_fp32_matches_oracle_fresh_input(sd):
    imgs = synth_images(11, [(640, 640)])
    m = _model(sd, "fp32")
    proc = DETRProcessor(m.config, image_size=640)
    x, _ = proc.preprocess(imgs, device=m.device)
    taps, otaps = {}, {}
    out = m(x, taps=taps)
    with torch.no_grad():
        s, b = O.detr_forward(sd, O.detr_preprocess(imgs, (640, 640)), O.DetrOracleConfig(), otaps)
    ds, db = compare_queries(s.numpy(), b.numpy(), otaps["topk_ind"].numpy(), out.logits.cpu().numpy(), out.boxes.cpu().numpy(), taps["topk_ind"].cpu().numpy())
    _report("fp32_vs_oracle_fresh", {"scores_max_abs": ds, "boxes_max_abs": db})
    assert ds < 1e-3 and db < 1e-3


@pytest.mark.parametrize("algo,name", [(ops.ALGO_SIMT, "fp16_simt"), (ops.ALGO_AUTO, "fp16_tcgen05")])
def test_fp16_vs_reference_golden(sd, algo, name):
    g = load_golden("detr_l_obj365_b2_640")
    m = _model(sd, "fp16", algo)
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=m.device)
    taps = {}
    out = m(x, taps=taps)
    torch.cuda.synchronize()
    rel = {}
    for t in ("res3", "res4", "res5"):
        v = taps[t].permute(0, 3, 1, 2).float().cpu()
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        rel[t] = float(np.abs(sl - g["tap_" + t]).max() / g["tapstat_" + t][2])
    keys = taps["topk_ind"].cpu().numpy()
    overlap = _set_stats(g["enc_topk_ind"], keys)
    ds, db = _common_err(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.cpu().numpy(), out.boxes.cpu().numpy(), keys)
    dets = proc.postprocess(out, imgs, threshold=0.5)
    det_match = []
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        ref_set = set(zip(g["det_labels"][i, :n].tolist(), map(tuple, g["det_boxes"][i, :n].tolist())))
        got = set((x.cls_id, tuple(x.bbox)) for x in d.detections)
        det_match.append({"ref": n, "got": len(got), "exact_common": len(ref_set & got)})
    _report(name, {"backbone_rel_err": rel, "enc_query_overlap_of_300": overlap, "scores_max_abs_common": ds, "boxes_max_abs_common": db, "detections": det_match})
    assert all(v < 2e-2 for v in rel.values()), rel
    assert min(overlap) >= 240, overlap
    assert torch.isfinite(out.logits).all() and torch.isfinite(out.boxes).all()


def test_batch_invariance_and_full_size(sd):
    """BASELINE full size (B=32, 640²): size-independent properties — per-image results do not depend on the batch
    they were computed in (bit-exact), post-process output is sorted and idempotent w.r.t. its own keep-set."""
    m = _model(sd, "fp16")
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(21, [(640, 640)] * 32)
    x, _ = proc.preprocess(imgs, device=m.device)
    out32 = m(x)
    out4 = m(x[4:8].contiguous())
    assert torch.equal(out32.logits[4:8], out4.logits) and torch.equal(out32.boxes[4:8], out4.boxes)
    s, l, b, q, c = proc.postprocess_tensors(out32, [(640, 640)] * 32, threshold=0.5)
    assert bool((s[:, :-1] >= s[:, 1:]).all()), "sorted by descending score"
    assert bool(((s > 0.5).sum(1) == c).all())
    # the flat index (query*C + label) must point back at the same score
    flat = out32.logits.reshape(32, -1).gather(1, (q.long() * out32.logits.shape[-1] + l.long()))
    assert torch.equal(flat, s)


def test_fp32_tc_runs_the_pair_flow_and_meets_the_parity_bars(sd):
    """precision="fp32_tc" (split-precision tensor-core convs/linears, activations as fp16 [hi|lo] pairs between convs): same bars as the fp32 SIMT mode."""
    g = load_golden("detr_l_obj365_b2_640")
    m = _model(sd, "fp32_tc")
    proc = DETRProcessor(m.config, image_size=640)
    imgs = synth_images(1, [(640, 640)] * 2)
    x, _ = proc.preprocess(imgs, device=m.device)
    taps = {}
    trace = ops.enable_trace()
    try:
        out = m(x, taps=taps)
        torch.cuda.synchronize()
    finally:
        ops.enable_trace(False)
    symbols = [e[0] for e in trace]
    assert "fb200_conv2d_pair" in symbols and "fb200_conv2d" not in symbols, "every conv / linear of the fp32_tc flow runs as conv2d_pair"
    for t in ("res3", "res4", "res5"):
        v = taps[t].permute(0, 3, 1, 2).float().cpu()
        sl = v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()
        assert np.abs(sl - g["tap_" + t]).max() <= 2e-4 * g["tapstat_" + t][2], t
    keys = taps["topk_ind"].cpu().numpy()
    assert _set_stats(g["enc_topk_ind"], keys) == [300, 300], "encoder query SETS must be identical"
    ds, db = compare_queries(g["scores"], g["boxes"], g["enc_topk_ind"], out.logits.cpu().numpy(), out.boxes.cpu().numpy(), keys)
    _report("fp32_tc_vs_reference_golden", {"scores_max_abs": ds, "boxes_max_abs": db})
    assert ds < 1e-3 and db < 1e-3, (ds, db)
    dets = proc.postprocess(out, imgs, threshold=0.5)
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert sorted(x.cls_id for x in d.detections) == sorted(g["det_labels"][i, :n].tolist())
        assert sorted(tuple(x.bbox) for x in d.detections) == sorted(map(tuple, g["det_boxes"][i, :n].tolist()))


def test_focoos_model_cuda_graph_path_equals_eager(sd):
    """FocoosModel replays a captured CUDA graph of model.forward from the second sighting of an input shape: identical detections, call after call,
    also with different images flowing through the same static buffers."""
    from focoos_b200 import FocoosModel, ModelInfo

    fm = FocoosModel(_model(sd, "fp32"), ModelInfo(name="fai-detr-l-obj365", im_size=640))
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
    """FocoosModel.infer_async / stream (copy stream + two staging buffers + pinned result buffers): same detections as the blocking call, for
    different images flowing through the same buffers, in order."""
    from focoos_b200 import FocoosModel, ModelInfo

    fm = FocoosModel(_model(sd, "fp16"), ModelInfo(name="fai-detr-l-obj365", im_size=640))
    batches = [torch.from_numpy(np.stack(synth_images(s, [(640, 640)] * 2))).pin_memory() for s in (1, 2, 3, 4, 5)]
    ref = [fm(b, threshold=0.5, batched=True) for b in batches]
    key = lambda dets: [[(d.cls_id, tuple(d.bbox), d.conf) for d in x.detections] for x in dets]
    got = list(fm.stream(batches, threshold=0.5))
    assert [key(g) for g in got] == [key(r) for r in ref]
    # a handle may be resolved late (its pinned buffer is only reused two submissions later) and twice
    h1 = fm.infer_async(batches[0], threshold=0.5)
    h2 = fm.infer_async(batches[1], threshold=0.5)
    assert key(h2.result()) == key(ref[1]) and key(h1.result()) == key(ref[0]) and key(h1.result()) == key(ref[0])
    # non-pinned / list inputs fall back to the synchronous path
    assert key(fm.infer_async([b for b in batches[2].numpy()], threshold=0.5).result()) == key(ref[2])


def test_export_roundtrip_on_gpu(sd, tmp_path):
    """FocoosModel.export on the GPU: the TorchScript file (one focoos_b200::model_forward op over its own weights) reloads and reproduces the eager
    tensors bit for bit, in the parity-green tensor-core mode; the exported InferModel returns the same detections as FocoosModel.infer."""
    from focoos_b200 import FocoosModel, ModelInfo

    fm = FocoosModel(_model(sd, "fp32_tc"), ModelInfo(name="fai-detr-l-obj365", im_size=640))
    im = fm.export(out_dir=str(tmp_path), image_size=640)
    x = 128 * torch.randn(2, 3, 640, 640, device="cuda")
    eager = fm.model(x)
    loaded = torch.jit.load(str(tmp_path / "model.pt"))
    boxes, logits = loaded(x)
    assert torch.equal(boxes, eager.boxes) and torch.equal(logits, eager.logits)
    img = synth_images(31, [(480, 600)])[0]
    d1, d2 = im.infer(img, threshold=0.5), fm.infer(img, threshold=0.5)
    assert [(d.cls_id, d.bbox, d.conf) for d in d1.detections] == [(d.cls_id, d.bbox, d.conf) for d in d2.detections]
