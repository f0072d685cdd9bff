"""Box-AP evaluation on the GPU: the matching kernel against BoxAPEvaluator's matching loop on the edge cases and at full size, its refusals, model.eval
of the fai-detr models against BoxAPEvaluator on the same eval_postprocess outputs, and (with two GPUs) multi-GPU evaluation against one GPU."""
import numpy as np
import pytest
import torch

from focoos_b200 import ModelManager, ops
from focoos_b200.ports import Boxes, Instances
from focoos_b200.trainer import BoxAPEvaluator, DeviceBoxAPEvaluator, SyntheticDetectionDataset, SyntheticSemSegDataset, TrainerArgs, inference_on_dataset
from tests.test_box_ap_eval_cpu import THRS, evaluator_tp_bits, gt_arrays, make_case, padded

pytestmark = pytest.mark.gpu
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")


def _kernel(outputs, entries, C):
    s, c, b, counts = padded(outputs)
    gb, gc, off = gt_arrays(entries)
    npos = torch.zeros(C, dtype=torch.int64, device="cuda")
    tp = ops.box_ap_match(s.cuda(), c.cuda(), b.cuda(), torch.tensor(counts, dtype=torch.int32).cuda(), gb.cuda(), gc.cuda(), off, THRS, C, npos)
    got = tp.cpu().numpy().astype(np.int64) & 0xFFFF
    assert all((got[i, n:] == 0).all() for i, n in enumerate(counts)), "bits past the count are zero"
    return np.concatenate([got[i, :n] for i, n in enumerate(counts)]), npos.cpu().numpy(), gc.numpy()


def _full_case(seed, B, C=365, K=300, G=200, fp64=False):
    """eval_postprocess-sized batches: K = 300 detections per image over 365 classes, up to 200 ground truths, continuous coordinates with a quarter of
    the detections copied (and jittered by whole pixels) from ground truths; scores rounded to 1/64 (ties)"""
    rng = np.random.default_rng(seed)
    entries, outputs = [], []
    for b in range(B):
        ng = int(rng.integers(0, G + 1)) if b else G
        gxy = rng.random((ng, 2)) * 600
        gb = np.concatenate([gxy, gxy + 4 + rng.random((ng, 2)) * 120], 1)
        gc = rng.integers(0, 40, ng)  # a few classes, so that images hold many same-class ground truths
        dxy = rng.random((K, 2)) * 600
        db = np.concatenate([dxy, dxy + 4 + rng.random((K, 2)) * 120], 1)
        dc = rng.integers(0, 40, K)
        if ng:
            src = rng.integers(0, ng, K // 4)
            db[: K // 4] = gb[src] + rng.integers(-3, 4, (K // 4, 4))
            dc[: K // 4] = gc[src]
        ds = np.round(rng.random(K) * 64) / 64
        g = torch.from_numpy(gb if fp64 else gb.astype(np.float32))
        entries.append({"height": 640, "width": 640, "instances": {"boxes": g, "classes": torch.from_numpy(gc)}})
        outputs.append({"instances": Instances((640, 640), boxes=Boxes(torch.from_numpy(db.astype(np.float32))),
                                               scores=torch.from_numpy(ds.astype(np.float32)), classes=torch.from_numpy(dc))})
    return entries, outputs


@pytest.mark.parametrize("seed,fp64", [(0, False), (1, False), (2, True), (3, True), (4, False)])
def test_kernel_equals_the_evaluator_loop_on_edge_cases(seed, fp64):
    entries, outputs = make_case(seed, fp64=fp64)
    ev = BoxAPEvaluator(6)
    ev.process(entries, outputs)
    got, npos, gc = _kernel(outputs, entries, 6)
    assert np.array_equal(got, evaluator_tp_bits(ev)) and int(got[0]) == 1
    assert np.array_equal(npos, np.bincount(gc, minlength=6))


@pytest.mark.parametrize("B,fp64", [(1, False), (32, False), (32, True)])
def test_kernel_equals_the_evaluator_loop_at_full_size(B, fp64):
    entries, outputs = _full_case(B + int(fp64), B, fp64=fp64)
    ev = BoxAPEvaluator(365)
    ev.process(entries, outputs)
    want = evaluator_tp_bits(ev)
    got, npos, gc = _kernel(outputs, entries, 365)
    assert np.array_equal(got, want) and want.any()
    again, _, _ = _kernel(outputs, entries, 365)
    assert np.array_equal(again, got), "two runs are identical"
    assert np.array_equal(npos, np.bincount(gc, minlength=365))


def test_out_of_range_arguments_are_refused():
    dev = "cuda"
    s, c, b = torch.zeros((1, 8), device=dev), torch.zeros((1, 8), dtype=torch.int32, device=dev), torch.zeros((1, 8, 4), device=dev)
    cnt = torch.full((1,), 8, dtype=torch.int32, device=dev)
    npos = torch.zeros(4, dtype=torch.int64, device=dev)

    def call(s=s, c=c, b=b, cnt=cnt, G=3, off=None, thr=THRS):
        gb, gc = torch.zeros((G, 4), device=dev), torch.zeros(G, dtype=torch.int32, device=dev)
        off = torch.tensor([0, G] if off is None else off, dtype=torch.int32)
        return ops.box_ap_match(s, c, b, cnt, gb, gc, off, thr, 4, npos)

    call()
    big = 1025
    with pytest.raises(RuntimeError, match="1025 detections per image"):
        call(s=torch.zeros((1, big), device=dev), c=torch.zeros((1, big), dtype=torch.int32, device=dev), b=torch.zeros((1, big, 4), device=dev))
    with pytest.raises(RuntimeError, match="1025 ground truths"):
        call(G=1025)
    with pytest.raises(RuntimeError, match="not monotonic"):
        call(s=torch.zeros((2, 8), device=dev), c=torch.zeros((2, 8), dtype=torch.int32, device=dev), b=torch.zeros((2, 8, 4), device=dev),
             cnt=torch.zeros(2, dtype=torch.int32, device=dev), G=3, off=[0, 5, 3])
    with pytest.raises(RuntimeError, match="17 thresholds"):
        call(thr=np.linspace(0.1, 0.9, 17))
    torch.cuda.synchronize()
    assert npos.tolist() == [3, 0, 0, 0], "only the accepted call counted its ground truths: the refused ones launched nothing"


MODELS = [("fai-detr-l-obj365", 365), ("fai-detr-m-coco", 80)]


@pytest.mark.parametrize("name,C", MODELS)
@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
def test_model_eval_equals_the_host_evaluator(name, C, precision):
    """inference_on_dataset (DeviceBoxAPEvaluator) == BoxAPEvaluator over the same eval_postprocess outputs (top_k = 300)"""
    fm = ModelManager.get(name, precision=precision)
    data = SyntheticDetectionDataset(n=10, size=640, num_classes=C)
    ev, dev = BoxAPEvaluator(C), DeviceBoxAPEvaluator(C)
    for s in range(0, 10, 4):
        entries = [data[i] for i in range(s, min(10, s + 4))]
        out = fm.model(torch.stack([e["image"] for e in entries]).cuda().float())
        pp = fm.processor.eval_postprocess(out, entries, None)
        ev.process(entries, pp)
        dev.process(entries, pp)
    want = ev.evaluate()
    assert dev.evaluate() == want and want["num_detections"] == 3000 and want["num_images"] == 10
    assert inference_on_dataset(fm, data, batch_size=4) == want


# ---- two GPUs: each rank forwards whole batches of the one-GPU run (the dataset is a multiple of 2 x batch), so the model arithmetic is the same ----------
@two_gpus
def test_two_gpu_model_eval_equals_one_gpu(tmp_path):
    fm = ModelManager.get("fai-detr-l-obj365")
    data = SyntheticDetectionDataset(n=8, size=640, num_classes=365)
    one = fm.eval(TrainerArgs(run_name="one", output_dir=str(tmp_path), batch_size=2, num_gpus=1), data, save_json=False)
    two = fm.eval(TrainerArgs(run_name="two", output_dir=str(tmp_path), batch_size=2, num_gpus=2, master_port=29561), data, save_json=True)
    assert two == one and one["num_images"] == 8 and (tmp_path / "two" / "eval_metrics.json").exists()
    seg = ModelManager.get("bisenetformer-s-ade")
    sdata = SyntheticSemSegDataset(n=8, sizes=((357, 483), (250, 333)))
    one = seg.eval(TrainerArgs(run_name="s1", output_dir=str(tmp_path), batch_size=2, num_gpus=1), sdata, save_json=False)
    two = seg.eval(TrainerArgs(run_name="s2", output_dir=str(tmp_path), batch_size=2, num_gpus=2, master_port=29562), sdata, save_json=False)
    assert two == one and one["sem_seg"]["pACC"] is not None


@two_gpus
def test_two_gpu_training_reports_metrics_of_all_validation_data(tmp_path):
    fm = ModelManager.get("fai-detr-l-obj365")
    data = SyntheticDetectionDataset(n=8, size=640, num_classes=365)
    val = SyntheticDetectionDataset(n=4, size=640, num_classes=365, seed=9)
    args = TrainerArgs(run_name="t", output_dir=str(tmp_path), num_gpus=2, max_iters=2, batch_size=2, log_period=1, master_port=29563)
    info = fm.train(args, data, data_val=val)
    assert info["val_metrics"]["num_images"] == 4
    assert inference_on_dataset(fm, val, batch_size=2) == info["val_metrics"], "the trained weights evaluated on one GPU over all of data_val"
