"""Box-AP evaluation on the device without a GPU: the CPU operator of the matching kernel (oracle/box_ap_ref.py) against BoxAPEvaluator's matching loop,
DeviceBoxAPEvaluator against BoxAPEvaluator, two gloo ranks against one for the box and semantic evaluators, and periodic evaluation while
fine-tuning (eval_period) without an effect on the trained weights."""
import math
import os
import pickle
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from focoos_b200 import ops
from focoos_b200.ports import Boxes, Instances
from focoos_b200.trainer import (BoxAPEvaluator, DeviceBoxAPEvaluator, SemSegEvaluator, SyntheticDetectionDataset, SyntheticSemSegDataset, TrainerArgs,
                                 _iou_matrix, inference_on_dataset)
from oracle.box_ap_ref import BoxAPRefBackend

THRS = np.arange(0.5, 0.96, 0.05)


@pytest.fixture()
def ref_backend():
    ops._backend = BoxAPRefBackend()
    yield
    ops._backend = None


def evaluator_tp_bits(ev: BoxAPEvaluator) -> np.ndarray:
    """the true-positive bits of every detection of ev.dets (in its order) as BoxAPEvaluator.evaluate's loop assigns them (same statements)"""
    bits = np.zeros(len(ev.dets), dtype=np.int64)
    for c in range(ev.num_classes):
        gts = {k[0]: np.stack(v) for k, v in ev.gts.items() if k[1] == c}
        if sum(len(v) for v in gts.values()) == 0:
            continue
        pos = sorted((i for i, d in enumerate(ev.dets) if d[1] == c), key=lambda i: -ev.dets[i][2])
        dets = [ev.dets[i] for i in pos]
        ious = [(_iou_matrix(d[3][None], gts[d[0]])[0] if d[0] in gts else np.zeros(0)) for d in dets]
        for ti, t in enumerate(THRS):
            used = {k: np.zeros(len(v), dtype=bool) for k, v in gts.items()}
            for di, d in enumerate(dets):
                iou = ious[di]
                if iou.size:
                    cand = np.where(used[d[0]], -1.0, iou)
                    j = int(cand.argmax())
                    if cand[j] >= t:
                        used[d[0]][j] = True
                        bits[pos[di]] |= 1 << ti
    return bits


def make_case(seed: int, B: int = 5, K: int = 40, G: int = 14, C: int = 6, fp64: bool = False):
    """(entries with ground truth, eval_postprocess-like outputs) on an integer grid, so that IoUs land exactly on thresholds and tie: scores from four
    values (ties inside and across images), a duplicated ground truth (two tied for the best IoU), image 1 without ground truth, image 2 without
    detections, class C-1 without ground truth, image 0 holding [0,0,2,1] against [0,0,1,1] (IoU exactly 0.5)"""
    rng = np.random.default_rng(seed)
    entries, outputs = [], []
    for b in range(B):
        ng = 0 if b == 1 else int(rng.integers(2, G + 1))
        gxy = rng.integers(0, 6, (ng, 2))
        gb = np.concatenate([gxy, gxy + rng.integers(1, 4, (ng, 2))], 1).astype(np.float64)
        gc = rng.integers(0, C - 1, ng)
        if ng >= 2:
            gb[1], gc[1] = gb[0], gc[0]
        nd = 0 if b == 2 else int(rng.integers(1, K + 1))
        near = gb[rng.integers(0, ng, nd)] + rng.integers(-1, 2, (nd, 4)) * 0.5 if ng else np.zeros((nd, 4))
        dxy = rng.integers(0, 6, (nd, 2))
        rand = np.concatenate([dxy, dxy + rng.integers(1, 4, (nd, 2))], 1)
        db = np.where(rng.random((nd, 1)) < 0.7, near, rand)
        db[:, 2:] = np.maximum(db[:, 2:], db[:, :2] + 0.5)
        dc = np.where(rng.random(nd) < 0.7, gc[rng.integers(0, ng, nd)] if ng else 0, rng.integers(0, C, nd))
        ds = rng.choice(np.array([0.9, 0.5, 0.25, 0.125], np.float32), nd)
        if b == 0:
            gb[0], db[0], dc[0], ds[0] = [0, 0, 1, 1], [0, 0, 2, 1], gc[0], 1.0
        g = torch.from_numpy(gb if fp64 else gb.astype(np.float32))
        entries.append({"height": 8, "width": 8, "instances": {"boxes": g, "classes": torch.from_numpy(gc)}})
        outputs.append({"instances": Instances((8, 8), boxes=Boxes(torch.from_numpy(db.astype(np.float32))), scores=torch.from_numpy(ds),
                                               classes=torch.from_numpy(dc.astype(np.int64)))})
    return entries, outputs


def padded(outputs):
    B = len(outputs)
    counts = [len(o["instances"].scores) for o in outputs]
    K = max(max(counts), 1)
    s, c, b = torch.zeros((B, K)), torch.full((B, K), -1, dtype=torch.int32), torch.zeros((B, K, 4))
    for i, o in enumerate(outputs):
        n = counts[i]
        s[i, :n], c[i, :n], b[i, :n] = o["instances"].scores, o["instances"].classes.int(), o["instances"].boxes.tensor
    return s, c, b, counts


def gt_arrays(entries):
    gb = torch.cat([e["instances"]["boxes"] for e in entries])
    gc = torch.cat([e["instances"]["classes"] for e in entries]).int()
    off = torch.tensor([0] + np.cumsum([len(e["instances"]["classes"]) for e in entries]).tolist(), dtype=torch.int32)
    return gb, gc, off


def same(a: dict, b: dict) -> bool:
    """dict equality with NaN equal to NaN (the no-ground-truth branch)"""
    if a == b:
        return True
    return repr(a) == repr(b) and any(isinstance(v, float) and math.isnan(v) for v in a.get("bbox", {}).values())


@pytest.mark.parametrize("seed,fp64", [(0, False), (1, False), (2, True), (3, True), (4, False)])
def test_reference_matching_equals_the_evaluator_loop(seed, fp64):
    entries, outputs = make_case(seed, fp64=fp64)
    ev = BoxAPEvaluator(6)
    ev.process(entries, outputs)
    want = evaluator_tp_bits(ev)
    s, c, b, counts = padded(outputs)
    gb, gc, off = gt_arrays(entries)
    npos = torch.zeros(6, dtype=torch.int64)
    ops._backend = BoxAPRefBackend()
    try:
        tp = ops.box_ap_match(s, c, b, torch.tensor(counts, dtype=torch.int32), gb, gc, off, THRS, 6, npos)
    finally:
        ops._backend = None
    got = np.concatenate([tp[i, :n].numpy().astype(np.int64) & 0xFFFF for i, n in enumerate(counts)])
    assert np.array_equal(got, want)
    assert want.any() and (want != (1 << len(THRS)) - 1).any(), "the case has hits and misses"
    assert int(want[0]) == 1, "IoU exactly 0.5: a hit at 0.50 only"
    assert np.array_equal(npos.numpy(), np.bincount(gc.numpy(), minlength=6))


@pytest.mark.parametrize("seed,fp64,batches", [(0, False, [5]), (1, True, [2, 3]), (5, False, [1, 1, 3])])
def test_device_evaluator_equals_the_host_evaluator(ref_backend, seed, fp64, batches):
    entries, outputs = make_case(seed, fp64=fp64)
    ev, dev = BoxAPEvaluator(6), DeviceBoxAPEvaluator(6)
    s = 0
    for n in batches:
        ev.process(entries[s:s + n], outputs[s:s + n])
        dev.process(entries[s:s + n], outputs[s:s + n])
        s += n
    assert dev.evaluate() == ev.evaluate()


def test_device_evaluator_mixed_ground_truth_precision_and_empty_cases(ref_backend):
    e32, o32 = make_case(6)
    e64, o64 = make_case(7, fp64=True)
    entries, outputs = e32[:3] + e64[:3], o32[:3] + o64[:3]
    ev, dev = BoxAPEvaluator(6), DeviceBoxAPEvaluator(6)
    ev.process(entries, outputs)
    dev.process(entries, outputs)
    assert dev.evaluate() == ev.evaluate()
    for ents in ([], [{"height": 8, "width": 8}]):  # nothing processed; one image without ground truth or detections: the NaN branch
        outs = [{"instances": Instances((8, 8), boxes=Boxes(torch.zeros((0, 4))), scores=torch.zeros(0), classes=torch.zeros(0, dtype=torch.int64))}] * len(ents)
        ev.reset(), dev.reset()
        ev.process(ents, outs)
        dev.process(ents, outs)
        a, b = dev.evaluate(), ev.evaluate()
        assert same(a, b) and math.isnan(a["bbox"]["AP"]) and a["num_detections"] == 0


def test_inference_on_dataset_picks_the_device_evaluator(ref_backend):
    from tests.test_api_cpu import _fm
    fm = _fm(size=128, num_classes=5)
    data = SyntheticDetectionDataset(n=3, size=128, num_classes=5)
    got = inference_on_dataset(fm, data, batch_size=2)
    ev = BoxAPEvaluator(5)
    assert inference_on_dataset(fm, data, batch_size=2, evaluator=ev) == got and got["num_images"] == 3


# ---- two gloo ranks ---------------------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _sem_seg_scores(ds, i, C=150):
    """seeded [C,H,W] scores of entry i (ties from a coarse value set)"""
    H, W = ds[i]["sem_seg"].shape
    g = torch.Generator().manual_seed(1000 + i)
    return torch.randint(0, 6, (C, H, W), generator=g).float()


def _run_evaluations():
    """(box-AP dict of inference_on_dataset over 5 synthetic detection images, the semantic evaluator's (matrix, metrics) over 5 synthetic ADE entries),
    each rank of an initialised group taking its shard"""
    from focoos_b200 import distributed as D
    from tests.test_api_cpu import _fm
    ops._backend = BoxAPRefBackend()
    try:
        torch.manual_seed(0)  # the class head of a 5-class model is not in the seeded weights: the same initialisation in every process
        fm = _fm(size=128, num_classes=5)
        det = inference_on_dataset(fm, SyntheticDetectionDataset(n=5, size=128, num_classes=5), batch_size=1)  # per-image forwards: the same arithmetic on any shard
        ds = SyntheticSemSegDataset(n=5, sizes=((37, 45), (30, 41)))
        ev = SemSegEvaluator(150)
        ev.reset()
        lo, hi = D.shard_range(len(ds))
        from oracle.sem_seg_ref import SemSegRefBackend
        ops._backend = SemSegRefBackend()
        for i in range(lo, hi):
            ev.process([ds[i]], [{"sem_seg": _sem_seg_scores(ds, i)}])
        return det, ev.evaluate()
    finally:
        ops._backend = None


def _rank(rank, world, port, path):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = _run_evaluations()
    with open(f"{path}.{rank}", "wb") as f:
        pickle.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


def test_two_gloo_ranks_equal_one(tmp_path):
    threads = torch.get_num_threads()
    torch.set_num_threads(2)  # as the ranks: the CPU operators' reductions depend on the thread count
    try:
        one = _run_evaluations()
    finally:
        torch.set_num_threads(threads)
    assert one[0]["num_images"] == 5 and one[1]["sem_seg"]["mIoU"] is not None
    path = str(tmp_path / "res")
    mp.start_processes(_rank, args=(2, _free_port(), path), nprocs=2, join=True, start_method="spawn")
    with open(f"{path}.0", "rb") as f:
        r0 = pickle.load(f)
    with open(f"{path}.1", "rb") as f:
        r1 = pickle.load(f)
    assert r0 == one, "rank 0 reports the whole dataset, exactly"
    assert r1 == ({}, {}), "the other ranks return {}"


# ---- eval_period ------------------------------------------------------------------------------------------------------------------------------------
def test_eval_period_logs_where_eval_hook_would_and_does_not_touch_training(ref_backend, tmp_path):
    from tests.test_api_cpu import _fm
    data = SyntheticDetectionDataset(n=4, size=128, num_classes=5)
    val = SyntheticDetectionDataset(n=3, size=128, num_classes=5, seed=9)
    runs = {}
    for period in (0, 1):
        torch.manual_seed(0)  # the same initial weights (the 5-class head is not in the seeded weights)
        fm = _fm(size=128, num_classes=5)
        args = TrainerArgs(run_name=f"p{period}", output_dir=str(tmp_path), num_gpus=1, max_iters=2, batch_size=2, log_period=1, eval_period=period)
        info = fm.train(args, data, data_val=val)
        runs[period] = (info, {k: v.clone() for k, v in fm.model.state_dict().items()})
    (info0, sd0), (info1, sd1) = runs[0], runs[1]
    assert all(torch.equal(sd0[k], sd1[k]) for k in sd0), "periodic evaluation leaves the trained weights and buffers bit-identical"
    evals = [h for h in info1["training_history"] if "val_metrics" in h]
    assert [h["iter"] for h in evals] == [0, 1], "after iteration 0 (1 % 1 == 0, not the last) and once after the last"
    assert evals[-1]["val_metrics"] == info1["val_metrics"] == info0["val_metrics"]
    assert [h for h in info1["training_history"] if "val_metrics" not in h] == info0["training_history"], "the loss log is unchanged"
    assert not any("val_metrics" in h for h in info0["training_history"])
    assert set(info1["val_metrics"]["bbox"]) == {"AP", "AP50", "AP75"} and info1["val_metrics"]["num_images"] == 3
