"""`FocoosModel.train` / `FocoosModel.eval` for the fai-detr family — the slice of the reference's trainer that sits ON the hot path
(SURVEY §3.3/§3.5, §8 a21/f3):

  TrainerLoop.run_step              focoos/trainer/trainer.py:723-773      -> train_step.TrainStep (forward, criterion, backward, exchange, AdamW)
  DETRProcessor.preprocess (train)  focoos/models/fai_detr/processor.py:66-100 -> `training_batch` below (DatasetEntry list -> images + DETRTargets)
  WarmupMultiStepLR                 focoos/trainer/solver/lr_scheduler.py:73-110 -> `lr_factor`
  run_train / launch                focoos/trainer/trainer.py:283-420, utils/distributed/dist.py:40-137 -> `run_train_entry` (one process per GPU, NCCL)
  inference_on_dataset              focoos/trainer/evaluation/evaluator.py:115-238 -> `inference_on_dataset` (batched, instances stay on the device)
  EMAHook / EMAUpdater              focoos/trainer/solver/ema.py:96-228    -> train_step.ModelEMA (TrainerArgs.ema_enabled: one device pass per step,
                                                                              evaluation and model_final.pth from the averaged weights)

Out of scope (reference control plane, SURVEY §2): hooks, checkpointer rotation, resume / init_checkpoint (so no `ema_state` in checkpoints, and
`ema_warmup` applies as given), Hub sync, tensorboard, COCO-json evaluators (pycocotools);
`BoxAPEvaluator` below is a small self-contained AP@[.5:.95] / AP50 so that `model.eval` returns numbers without those dependencies.

Dataset contract (reference `MapDataset` of `DatasetEntry`, ports.py): `len(ds)`, `ds[i]` -> entry with `.image` (uint8 / float tensor [3,H,W]),
`.height`, `.width`, `.instances` with `.boxes.tensor` ([n,4] absolute xyxy in the image's pixels) and `.classes` ([n] int64); plain dicts with the
same keys are accepted.  Images of one batch must share one size that is a multiple of 32 (the reference pads with ImageList; the synthetic
COCO-shape data of BASELINE configs[4] is 640x640).
"""
from __future__ import annotations

import contextlib
import json
import os
from dataclasses import asdict, dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist

from . import distributed as D
from . import ops
from .criterion import DETRTargets
from .ports import Boxes, Instances


@dataclass
class TrainerArgs:
    """ports.py:973-1066 — the fields the hot path reads (same names and defaults)."""

    run_name: str
    output_dir: str = os.path.join(os.path.expanduser("~"), "FocoosAI", "models")
    num_gpus: int = 1
    device: str = "cuda"
    amp_enabled: bool = True
    eval_period: int = 0
    log_period: int = 20
    seed: int = 42
    learning_rate: float = 5e-4
    weight_decay: float = 0.02
    max_iters: int = 3000
    batch_size: int = 16
    scheduler: str = "MULTISTEP"
    scheduler_extra: Optional[dict] = None
    optimizer: str = "ADAMW"
    weight_decay_norm: float = 0.0
    weight_decay_embed: float = 0.0
    backbone_multiplier: float = 0.1
    decoder_multiplier: float = 1.0
    head_multiplier: float = 1.0
    freeze_bn: bool = False
    clip_gradients: float = 0.1
    sync_bn: bool = True  # torch.nn.SyncBatchNorm.convert_sync_batchnorm when world_size > 1 (trainer.py:334)
    ema_enabled: bool = False  # model EMA (trainer.py:488-495): evaluation and model_final.pth from the averaged weights
    ema_decay: float = 0.999
    ema_warmup: int = 2000
    master_port: int = 29531


def _get(e, name):
    return e[name] if isinstance(e, dict) else getattr(e, name)


def training_batch(entries: Sequence, device) -> tuple:
    """fai_detr/processor.py:82-100: images stacked to [B,3,H,W] float (0..255), targets = DETRTargets(labels, boxes cxcywh normalised by the batch size)."""
    imgs = [_get(e, "image") for e in entries]
    assert all(tuple(i.shape) == tuple(imgs[0].shape) for i in imgs), "one image size per batch (multiple of 32)"
    x = torch.stack([i if torch.is_tensor(i) else torch.from_numpy(np.asarray(i)) for i in imgs]).to(device, non_blocking=True).float()
    h, w = x.shape[-2:]
    scale = torch.tensor([w, h, w, h], dtype=torch.float32, device=device)
    targets = []
    for e in entries:
        inst = _get(e, "instances")
        boxes = _get(inst, "boxes")
        bt = (boxes.tensor if hasattr(boxes, "tensor") else torch.as_tensor(boxes)).to(device).float() / scale
        cxcywh = torch.stack([(bt[:, 0] + bt[:, 2]) / 2, (bt[:, 1] + bt[:, 3]) / 2, bt[:, 2] - bt[:, 0], bt[:, 3] - bt[:, 1]], -1)  # utils/box.py:20-24
        targets.append(DETRTargets(labels=torch.as_tensor(_get(inst, "classes")).to(device).long(), boxes=cxcywh))
    return x, targets


def lr_factor(it: int, max_iters: int, scheduler: str = "MULTISTEP", extra: Optional[dict] = None) -> float:
    """WarmupMultiStepLR / cosine / poly of solver/lr_scheduler.py as a multiplicative factor on every group's base lr."""
    extra = dict(extra or {})
    warm_it, warm_f = int(extra.get("warmup_iters", 0)), float(extra.get("warmup_factor", 1.0))
    warm = 1.0
    if it < warm_it:
        a = it / max(1, warm_it)
        warm = warm_f * (1 - a) + a
    name = scheduler.upper()
    if name == "MULTISTEP":
        ms = [int(m * max_iters) for m in extra.get("milestones", [])]
        return warm * float(extra.get("gamma", 0.1)) ** sum(1 for m in ms if it >= m)
    if name == "COSINE":
        import math
        return warm * 0.5 * (1.0 + math.cos(math.pi * it / max_iters))
    if name == "POLY":
        return warm * (1.0 - it / max_iters) ** float(extra.get("power", 0.9))
    if name == "FIXED":
        return warm
    raise NotImplementedError(f"Scheduler {scheduler} is not supported")


def _train_worker(rank: int, world: int, fm, args: TrainerArgs, data_train, data_val, out_dir: str):
    from .train_step import FlatAdamW, GradBucketReducer, ModelEMA, TrainStep, get_optimizer_params
    if world > 1:
        os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(args.master_port))
        torch.cuda.set_device(rank)
        D.init_from_env("nccl", torch.device("cuda", rank))
    if ops._backend is not None:  # tests: host logic on the CPU reference operators (host tensors only)
        dev = torch.device("cpu")
    else:
        dev = torch.device("cuda", rank if world > 1 else torch.cuda.current_device())
    model = fm.model.to(dev)
    model.train()
    if args.freeze_bn and hasattr(model, "freeze_bn"):
        model.freeze_bn = True
    if hasattr(model, "sync_bn"):
        model.sync_bn = bool(args.sync_bn) and world > 1
    if hasattr(model, "train_precision") and model.train_precision is None and getattr(model, "precision", "fp32") != "fp32" and dev.type == "cuda":
        # TrainerArgs.amp_enabled (ports.py:1029, default True): the reference's iteration runs under torch.autocast(fp16) + GradScaler -> one fp16 tensor-core product
        # per conv/linear here; amp_enabled=False: fp32-accurate (three-product) arithmetic
        model.train_precision = "amp" if args.amp_enabled else "fp32_tc"
    opt = FlatAdamW(get_optimizer_params(model, args.learning_rate, args.weight_decay, args.weight_decay_norm, args.weight_decay_embed, args.backbone_multiplier,
                                         args.decoder_multiplier, args.head_multiplier), clip_gradients=args.clip_gradients, amp=args.amp_enabled, world_size=world)
    opt.track_unused_parameters()
    red = GradBucketReducer(opt)
    red.attach_hooks()
    # EMAHook.before_train: the EMA starts from the weights every rank trains from (after the reducer's broadcast); every rank keeps its own
    ema = ModelEMA(model, opt, args.ema_decay, args.ema_warmup) if args.ema_enabled else None
    step = TrainStep(model, opt, red, ema)
    g = torch.Generator().manual_seed(args.seed + rank)
    n = len(data_train)
    history = []
    for it in range(args.max_iters):
        idx = torch.randint(0, n, (args.batch_size,), generator=g).tolist()  # TrainingSampler: infinite shuffled stream, a different shard per rank
        x, targets = training_batch([data_train[i] for i in idx], dev)
        losses = step(x, targets, lr_factor(it, args.max_iters, args.scheduler, args.scheduler_extra))
        if args.log_period and (it % args.log_period == 0 or it == args.max_iters - 1):
            tot = float(sum(v.detach() for v in losses.values()))
            history.append({"iter": it, "total_loss": tot, **opt.stats()})
            if rank == 0:
                print(f"[focoos_b200.train] iter {it}: total_loss {tot:.4f} lr_factor {lr_factor(it, args.max_iters, args.scheduler, args.scheduler_extra):.3g} scale {history[-1]['scale']:.0f}", flush=True)
        # EvalHook.after_step (trainer/hooks/hook.py:539-545): every eval_period iterations; the one after the last iteration is the final evaluation
        if data_val is not None and args.eval_period > 0 and (it + 1) % args.eval_period == 0 and it + 1 != args.max_iters:
            history.append({"iter": it, "val_metrics": _evaluate_while_training(fm, data_val, args.batch_size, dev, ema)})
    if ema is not None:  # _store_model (trainer.py:367-375): the final evaluation and model_final.pth see the averaged weights
        ema.apply()
    metrics = None
    if data_val is not None:  # every rank evaluates its shard; rank 0 gets the metrics of all of data_val
        metrics = _evaluate_while_training(fm, data_val, args.batch_size, dev)
        if args.eval_period > 0:  # EvalHook.after_train
            history.append({"iter": args.max_iters - 1, "val_metrics": metrics})
    if rank == 0:
        os.makedirs(out_dir, exist_ok=True)
        torch.save({"model": {k: v.detach().cpu() for k, v in model.state_dict().items()}}, os.path.join(out_dir, "model_final.pth"))  # ArtifactName.WEIGHTS
        info = asdict(fm.model_info)
        info.update(weights_uri=os.path.join(out_dir, "model_final.pth"), val_metrics=metrics, train_args={k: v for k, v in asdict(args).items()}, training_history=history)
        with open(os.path.join(out_dir, "model_info.json"), "w") as f:  # ArtifactName.INFO
            json.dump(info, f, indent=1, default=str)
    red.detach_hooks()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _evaluate_while_training(fm, data_val, batch_size: int, dev, ema=None) -> dict:
    """inference_on_dataset between training iterations, leaving training as it was: no gradients flow (no_grad), the parameters, optimiser state and
    BatchNorm running statistics are only read (the eval forward packs its own copy of the weights), the global RNG state is restored, and the model
    returns to train mode.  With a ModelEMA the model holds the averaged weights during the evaluation and its training values again after it
    (apply_model_ema_and_restore, trainer.py:447-452); the eval engine is packed afresh from them, as model.eval() drops the packed one.
    {} on ranks other than 0."""
    model = fm.model
    with torch.random.fork_rng(devices=[dev] if dev.type == "cuda" else []), (ema.applied() if ema is not None else contextlib.nullcontext()):
        model.eval()
        try:
            return inference_on_dataset(fm, data_val, batch_size=batch_size)
        finally:
            model.train()


def run_train_entry(fm, args: TrainerArgs, data_train, data_val=None):
    assert args.num_gpus, "Training without GPUs is not supported. num_gpus must be greater than 0"  # focoos_model.py:249
    if type(fm.model).__name__ != "FAIDetr":
        raise NotImplementedError("focoos_b200 fine-tunes the fai-detr family (the segmentation families run inference only)")
    fm.model.check_trainable()
    out_dir = os.path.join(args.output_dir, args.run_name)
    if args.num_gpus > 1:
        import torch.multiprocessing as mp
        fm.model.cpu()
        fm._graphs.clear()
        fm._pipe = None
        mp.start_processes(_train_worker, args=(args.num_gpus, fm, args, data_train, data_val, out_dir), nprocs=args.num_gpus, join=True, start_method="spawn")
    else:
        _train_worker(0, 1, fm, args, data_train, data_val, out_dir)
    path = os.path.join(out_dir, "model_final.pth")
    if not os.path.exists(path):
        raise FileNotFoundError(f"Training did not end correctly, model file not found at {path}")  # focoos_model.py:265
    fm.model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True))
    if torch.cuda.is_available() and ops._backend is None:
        fm.model.cuda()
    fm.model.eval()
    fm.processor.eval()
    fm._graphs.clear()
    with open(os.path.join(out_dir, "model_info.json")) as f:
        return json.load(f)


# ---- evaluation ------------------------------------------------------------------------------------------------------------------------------
def _iou_matrix(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    lt = np.maximum(a[:, None, :2], b[None, :, :2])
    rb = np.minimum(a[:, None, 2:], b[None, :, 2:])
    inter = np.clip(rb - lt, 0, None).prod(-1)
    aa = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    ab = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    return inter / np.maximum(aa[:, None] + ab[None, :] - inter, 1e-12)


class BoxAPEvaluator:
    """process(inputs, outputs) / evaluate() like the reference's DatasetEvaluator (trainer/evaluation/evaluator.py:22-60): 101-point interpolated AP per class
    at IoU .50:.05:.95 (greedy matching in descending score order), averaged over the classes that have ground truth -> {"bbox": {"AP", "AP50", "AP75"}}."""

    def __init__(self, num_classes: int):
        self.num_classes = num_classes
        self.reset()

    def reset(self):
        self.dets: List[tuple] = []   # (image id, class, score, box)
        self.gts: Dict[tuple, List[np.ndarray]] = {}
        self._img = 0

    def process(self, inputs, outputs):
        for e, o in zip(inputs, outputs):
            inst = o["instances"]
            b, s, c = inst.boxes.tensor.cpu().numpy(), inst.scores.cpu().numpy(), inst.classes.cpu().numpy()
            for i in range(len(s)):
                self.dets.append((self._img, int(c[i]), float(s[i]), b[i]))
            gi = _get(e, "instances") if (isinstance(e, dict) and "instances" in e) or hasattr(e, "instances") else None
            if gi is not None:
                gb = _get(gi, "boxes")
                gb = (gb.tensor if hasattr(gb, "tensor") else torch.as_tensor(gb)).cpu().numpy().reshape(-1, 4)
                for box, cls in zip(gb, torch.as_tensor(_get(gi, "classes")).cpu().numpy().tolist()):
                    self.gts.setdefault((self._img, int(cls)), []).append(box)
            self._img += 1

    def evaluate(self):
        thrs = np.arange(0.5, 0.96, 0.05)
        aps = np.zeros((len(thrs), self.num_classes))
        has = np.zeros(self.num_classes, dtype=bool)
        for c in range(self.num_classes):
            gts = {k[0]: np.stack(v) for k, v in self.gts.items() if k[1] == c}
            npos = sum(len(v) for v in gts.values())
            if npos == 0:
                continue
            has[c] = True
            dets = sorted((d for d in self.dets if d[1] == c), key=lambda d: -d[2])
            ious = [(_iou_matrix(d[3][None], gts[d[0]])[0] if d[0] in gts else np.zeros(0)) for d in dets]
            for ti, t in enumerate(thrs):
                used = {k: np.zeros(len(v), dtype=bool) for k, v in gts.items()}
                tp = np.zeros(len(dets))
                for di, d in enumerate(dets):
                    iou = ious[di]
                    if iou.size:
                        cand = np.where(used[d[0]], -1.0, iou)
                        j = int(cand.argmax())
                        if cand[j] >= t:
                            used[d[0]][j] = True
                            tp[di] = 1
                ctp = np.cumsum(tp)
                rec = ctp / npos
                prec = ctp / np.maximum(np.arange(1, len(dets) + 1), 1)
                for i in range(len(prec) - 1, 0, -1):
                    prec[i - 1] = max(prec[i - 1], prec[i])
                rs = np.linspace(0, 1, 101)
                idx = np.searchsorted(rec, rs, side="left")
                aps[ti, c] = np.mean([prec[i] if i < len(prec) else 0.0 for i in idx]) if len(dets) else 0.0
        if not has.any():
            return {"bbox": {"AP": float("nan"), "AP50": float("nan"), "AP75": float("nan")}, "num_detections": len(self.dets)}
        return {"bbox": {"AP": float(aps[:, has].mean() * 100), "AP50": float(aps[0, has].mean() * 100), "AP75": float(aps[5, has].mean() * 100)},
                "num_detections": len(self.dets), "num_images": self._img}


class DeviceBoxAPEvaluator(BoxAPEvaluator):
    """BoxAPEvaluator with the matching on the device and the ranks combined; `evaluate` returns the dict BoxAPEvaluator returns for the same images.
    `process` runs the greedy matching of a whole batch in one launch (ops.box_ap_match) and keeps one record per detection on the device: score,
    class, true-positive bits per IoU threshold, image and detection index.  `evaluate` gathers the records of every rank (images numbered in rank
    order, as the contiguous shards of inference_on_dataset lie in the dataset), sums the ground-truth counts, and on rank 0 accumulates precision /
    recall per class in numpy: one stable sort by (class, -score, image, detection), cumulative sums, the precision envelope and the 101 recall points,
    with BoxAPEvaluator's arithmetic.  Other ranks return {} (as the reference's evaluators do)."""

    THRESHOLDS = np.arange(0.5, 0.96, 0.05)

    def reset(self):
        self._rec: List[torch.Tensor] = []  # int32 [n,5] per batch: score bits, class, tp bits, image (this rank), detection index
        self._npos = None                   # int64 [C] ground truths per class, on the device of the first batch
        self._img = 0
        self._ndet = 0

    @staticmethod
    def _gt(e):
        """(boxes [n,4] as the entry holds them, classes [n] int64) of an entry, as BoxAPEvaluator.process reads them"""
        gi = _get(e, "instances") if (isinstance(e, dict) and "instances" in e) or hasattr(e, "instances") else None
        if gi is None:
            return np.zeros((0, 4), np.float32), np.zeros((0,), np.int64)
        gb = _get(gi, "boxes")
        gb = (gb.tensor if hasattr(gb, "tensor") else torch.as_tensor(gb)).cpu().numpy().reshape(-1, 4)
        return gb, np.asarray(torch.as_tensor(_get(gi, "classes")).cpu().numpy(), dtype=np.int64).reshape(-1)

    def process(self, inputs, outputs):
        pairs = list(zip(inputs, outputs))
        if not pairs:
            return
        insts = [o["instances"] for _, o in pairs]
        dev = insts[0].scores.device
        B, C = len(pairs), self.num_classes
        counts = [int(i.scores.shape[0]) for i in insts]
        K = max(max(counts), 1)
        scores = torch.zeros((B, K), dtype=torch.float32, device=dev)
        classes = torch.full((B, K), -1, dtype=torch.int32, device=dev)
        boxes = torch.zeros((B, K, 4), dtype=torch.float32, device=dev)
        for b, (inst, n) in enumerate(zip(insts, counts)):
            scores[b, :n] = inst.scores
            classes[b, :n] = inst.classes
            boxes[b, :n] = inst.boxes.tensor
        gts = [self._gt(e) for e, _ in pairs]
        # numpy promotes the IoU of fp32 detections to fp64 for fp64 (or integer) ground truth: one launch per precision present in the batch
        fp64 = [np.result_type(np.float32, gb.dtype) == np.float64 for gb, _ in gts]
        if self._npos is None:
            self._npos = torch.zeros((C,), dtype=torch.int64, device=dev)
        tp = torch.zeros((B, K), dtype=torch.int16, device=dev)
        for prec in sorted(set(fp64)):
            sel = [b for b in range(B) if fp64[b] == prec]
            off = np.concatenate([[0], np.cumsum([len(gts[b][1]) for b in sel])]).astype(np.int32)
            gb = np.concatenate([gts[b][0] for b in sel]).astype(np.float64 if prec else np.float32).reshape(-1, 4)
            gc = np.clip(np.concatenate([gts[b][1] for b in sel]), -1, np.iinfo(np.int32).max).astype(np.int32)
            rows = slice(None) if len(sel) == B else torch.tensor(sel, device=dev)
            cnt = torch.tensor([counts[b] for b in sel], dtype=torch.int32).to(dev, non_blocking=True)
            t = ops.box_ap_match(scores[rows], classes[rows], boxes[rows], cnt, torch.from_numpy(gb).to(dev), torch.from_numpy(gc).to(dev),
                                 torch.from_numpy(off), self.THRESHOLDS, C, self._npos)
            tp[rows] = t
        rec = torch.stack([scores.view(torch.int32), classes, tp.to(torch.int32) & 0xFFFF,
                           (self._img + torch.arange(B, dtype=torch.int32, device=dev))[:, None].expand(B, K),
                           torch.arange(K, dtype=torch.int32, device=dev)[None, :].expand(B, K)], -1).reshape(B * K, 5)
        keep = np.concatenate([b * K + np.arange(n) for b, n in enumerate(counts)]).astype(np.int64)
        self._rec.append(rec.index_select(0, torch.from_numpy(keep).to(dev, non_blocking=True)))
        self._img += B
        self._ndet += sum(counts)

    def evaluate(self):
        C, T = self.num_classes, len(self.THRESHOLDS)
        rec = torch.cat(self._rec) if self._rec else torch.zeros((0, 5), dtype=torch.int32)
        parts = D.all_gather_rows(rec)
        imgs = D.gather_counts(self._img, D.collective_device())
        npos_t = torch.zeros((C,), dtype=torch.int64) if self._npos is None else self._npos
        npos = D.all_reduce_sum(npos_t).cpu().numpy()
        ndet = sum(D.gather_counts(self._ndet, D.collective_device()))
        if D.get_rank() != 0:
            return {}
        first = np.concatenate([[0], np.cumsum(imgs)[:-1]])
        R = np.concatenate([p.cpu().numpy() for p in parts]) if parts else np.zeros((0, 5), np.int32)
        img = R[:, 3].astype(np.int64) + np.repeat(first, [p.shape[0] for p in parts])
        score = np.ascontiguousarray(R[:, 0]).view(np.float32)
        cls, bits = R[:, 1], R[:, 2]
        order = np.lexsort((R[:, 4], img, -score.astype(np.float64), cls))
        cls, bits = cls[order], bits[order]
        aps = np.zeros((T, C))
        has = npos > 0
        rs = np.linspace(0, 1, 101)
        lo = np.searchsorted(cls, np.arange(C), side="left")
        hi = np.searchsorted(cls, np.arange(C), side="right")
        for c in np.nonzero(has)[0]:
            n = int(hi[c] - lo[c])
            if n == 0:
                continue
            tp = ((bits[lo[c]:hi[c]][None, :] >> np.arange(T)[:, None]) & 1).astype(np.float64)
            ctp = np.cumsum(tp, axis=1)
            recall = ctp / int(npos[c])
            prec = ctp / np.maximum(np.arange(1, n + 1), 1)
            prec = np.maximum.accumulate(prec[:, ::-1], axis=1)[:, ::-1]
            for ti in range(T):
                idx = np.searchsorted(recall[ti], rs, side="left")
                aps[ti, c] = np.mean(np.where(idx < n, prec[ti][np.minimum(idx, n - 1)], 0.0))
        if not has.any():
            return {"bbox": {"AP": float("nan"), "AP50": float("nan"), "AP75": float("nan")}, "num_detections": ndet}
        return {"bbox": {"AP": float(aps[:, has].mean() * 100), "AP50": float(aps[0, has].mean() * 100), "AP75": float(aps[5, has].mean() * 100)},
                "num_detections": ndet, "num_images": sum(imgs)}


def _box_ap_evaluator(num_classes: int) -> BoxAPEvaluator:
    """DeviceBoxAPEvaluator.  The host BoxAPEvaluator only when a test installs a CPU reference backend that does not restate the matching kernel
    (`ops._backend`; product code never sets it)."""
    if ops._backend is not None and not hasattr(ops._backend, "_box_ap_match"):
        return BoxAPEvaluator(num_classes)
    return DeviceBoxAPEvaluator(num_classes)


@torch.no_grad()
def inference_on_dataset(fm, dataset, batch_size: int = 16, evaluator=None, top_k: Optional[int] = None):
    """evaluator.py:115-238: run the model over `dataset` in batches (the reference uses batch 1 per GPU), `processor.eval_postprocess`, `evaluator.process`;
    each rank of an initialised process group takes a contiguous shard and the evaluator combines the ranks: rank 0 returns the metrics of the whole
    dataset, the other ranks {}.  The evaluator follows the processor: DeviceBoxAPEvaluator for DETRProcessor, SemSegEvaluator for MaskFormerProcessor,
    whose batches hold consecutive entries of one image size and run the model with `lazy_masks = True` (as FocoosModel.__call__ does)."""
    from .processor import MaskFormerProcessor
    model, proc = fm.model, fm.processor
    model.eval()
    if isinstance(proc, MaskFormerProcessor):
        return _sem_seg_inference(fm, dataset, batch_size, evaluator)
    evaluator = evaluator or _box_ap_evaluator(model.config.num_classes)
    evaluator.reset()
    lo, hi = D.shard_range(len(dataset))
    for s in range(lo, hi, batch_size):
        entries = [dataset[i] for i in range(s, min(hi, s + batch_size))]
        x = torch.stack([torch.as_tensor(_get(e, "image")) for e in entries]).to(model.device).float()
        out = model(x)
        evaluator.process(entries, proc.eval_postprocess(out, entries, top_k))
    return evaluator.evaluate()


def _sem_seg_inference(fm, dataset, batch_size, evaluator):
    model, proc = fm.model, fm.processor
    if evaluator is None:
        meta = getattr(dataset, "metadata", None)
        ignore = getattr(meta, "ignore_label", None)
        evaluator = SemSegEvaluator(model.config.num_classes, fm.model_info.classes, 255 if ignore is None else int(ignore))
    evaluator.reset()
    lo, hi = D.shard_range(len(dataset))
    s = lo
    while s < hi:
        entries = [dataset[s]]
        shape = tuple(torch.as_tensor(_get(entries[0], "image")).shape)
        while s + len(entries) < hi and len(entries) < batch_size:
            e = dataset[s + len(entries)]
            if tuple(torch.as_tensor(_get(e, "image")).shape) != shape:
                break
            entries.append(e)
        s += len(entries)
        x = torch.stack([torch.as_tensor(_get(e, "image")) for e in entries]).to(model.device).float()
        model.lazy_masks = True
        try:
            out = fm._forward(x)
        finally:
            model.lazy_masks = False
        evaluator.process(entries, proc.eval_postprocess(out, entries, precision=model.precision))
    return evaluator.evaluate()


def _eval_worker(rank: int, world: int, fm, args: TrainerArgs, data_test, result_path: str):
    """one rank of a multi-GPU model.eval: its shard through inference_on_dataset; rank 0 writes the metrics of the whole dataset to `result_path`"""
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(args.master_port))
    torch.cuda.set_device(rank)
    D.init_from_env("nccl", torch.device("cuda", rank))
    fm.model.cuda(rank)
    metrics = inference_on_dataset(fm, data_test, batch_size=args.batch_size)
    if rank == 0:
        with open(result_path, "w") as f:
            json.dump(metrics, f)
    dist.barrier()
    dist.destroy_process_group()


def run_eval_entry(fm, args: TrainerArgs, data_test, save_json: bool = True):
    """focoos_model.py:276-310: one process (num_gpus = 1) or one per GPU, each evaluating a contiguous shard, combined by the evaluator; the metrics of the
    whole dataset are returned, kept in model_info.val_metrics and written to <output_dir>/<run_name>/eval_metrics.json when `save_json`."""
    assert args.num_gpus, "Testing without GPUs is not supported. num_gpus must be greater than 0"  # focoos_model.py:300
    if args.num_gpus > 1:
        import tempfile

        import torch.multiprocessing as mp
        fm.model.cpu()
        fm._graphs.clear()
        fm._pipe = None
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "metrics.json")
            try:
                mp.start_processes(_eval_worker, args=(args.num_gpus, fm, args, data_test, path), nprocs=args.num_gpus, join=True, start_method="spawn")
            finally:
                fm.model.cuda()
            with open(path) as f:
                metrics = json.load(f)  # JSON keeps every float bit for bit (repr round trip), NaN included
    else:
        metrics = inference_on_dataset(fm, data_test, batch_size=args.batch_size)
    fm.model_info.val_metrics = metrics
    if save_json:
        out_dir = os.path.join(args.output_dir, args.run_name)
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "eval_metrics.json"), "w") as f:
            json.dump(metrics, f, indent=1)
    return metrics


def _sem_seg_gt(e) -> np.ndarray:
    """the entry's ground-truth label map [H,W]: `sem_seg` (array / tensor), or `sem_seg_file_name` read as load_image_into_numpy_array does
    (sem_seg_evaluation.py:28-34)"""
    if (isinstance(e, dict) and e.get("sem_seg") is not None) or getattr(e, "sem_seg", None) is not None:
        gt = _get(e, "sem_seg")
        return gt.cpu().numpy() if torch.is_tensor(gt) else np.asarray(gt)
    from PIL import Image
    with open(_get(e, "sem_seg_file_name"), "rb") as f:
        return np.array(Image.open(f))


class SemSegEvaluator:
    """SemSegEvaluator of trainer/evaluation/sem_seg_evaluation.py:37-163 with the reset / process / evaluate shape of BoxAPEvaluator.  `process` adds
    every image into a (C+1) x (C+1) int64 confusion matrix (row = predicted class, column = ground truth, ignore_label -> C) with one kernel launch
    (ops.sem_seg_confusion: argmax over the classes folded into the histogram); the matrix stays on the device until `evaluate`, which is the
    reference's numpy arithmetic -> {"sem_seg": {mIoU, fwIoU, IoU-<class>, mACC, pACC, ACC-<class>}}, non-finite values as None.  Class names are
    `class_names` when it names every class, the class indices otherwise."""

    def __init__(self, num_classes: int, class_names: Sequence[str] = (), ignore_label: int = 255):
        self.num_classes, self.ignore_label = num_classes, ignore_label
        self.class_names = list(class_names) if len(class_names) == num_classes else [str(i) for i in range(num_classes)]
        self.reset()

    def reset(self):
        self._conf = self._invalid = None  # allocated on the device of the first prediction

    def process(self, inputs, outputs):
        C = self.num_classes
        for e, o in zip(inputs, outputs):
            hwc = o["sem_seg"].permute(1, 2, 0)  # the NHWC score buffer eval_postprocess wrote
            if hwc.stride(-1) != 1:  # a [C,H,W] tensor that is not such a view
                hwc = hwc.contiguous()
            gt = _sem_seg_gt(e)
            assert gt.shape == tuple(hwc.shape[:2]), f"ground truth {gt.shape} vs prediction {tuple(hwc.shape[:2])}"
            if gt.dtype != np.uint8:  # int32 for the kernel; values beyond it stay out of [0, C] and are reported by evaluate()
                gt = np.clip(gt.astype(np.int64), -1, np.iinfo(np.int32).max).astype(np.int32)
            if self._conf is None:
                self._conf = torch.zeros((C + 1, C + 1), dtype=torch.int64, device=hwc.device)
                self._invalid = torch.zeros((1,), dtype=torch.int64, device=hwc.device)
            ops.sem_seg_confusion(hwc.unsqueeze(0), torch.from_numpy(np.ascontiguousarray(gt)).to(hwc.device, non_blocking=True).unsqueeze(0), C,
                                  self.ignore_label, self._conf, self._invalid)

    def confusion_matrix(self) -> np.ndarray:
        C = self.num_classes
        return np.zeros((C + 1, C + 1), dtype=np.int64) if self._conf is None else self._conf.cpu().numpy()

    def evaluate(self):
        """the metrics of this rank's matrix, or with a process group of several ranks, of the matrices summed over the ranks (on rank 0; {} elsewhere)"""
        if D.get_world_size() > 1:  # one SUM of [matrix | invalid count]; every rank raises on invalid labels
            C = self.num_classes
            local = torch.zeros(((C + 1) ** 2 + 1,), dtype=torch.int64)
            if self._conf is not None:
                local = torch.cat([self._conf.reshape(-1), self._invalid])
            tot = D.all_reduce_sum(local).cpu().numpy()
            conf, invalid = tot[:-1].reshape(C + 1, C + 1), int(tot[-1])
        else:
            conf, invalid = self.confusion_matrix(), 0 if self._invalid is None else int(self._invalid.item())
        if invalid:
            raise ValueError(f"{invalid} ground-truth pixels are neither in [0, {self.num_classes}] nor ignore_label={self.ignore_label}")
        if D.get_rank() != 0:
            return {}
        n = self.num_classes
        acc = np.full(n, np.nan, dtype=float)
        iou = np.full(n, np.nan, dtype=float)
        tp = conf.diagonal()[:-1].astype(float)
        pos_gt = np.sum(conf[:-1, :-1], axis=0).astype(float)
        with np.errstate(divide="ignore", invalid="ignore"):  # an empty matrix gives NaN metrics (None), as in the reference
            class_weights = pos_gt / np.sum(pos_gt)
            pos_pred = np.sum(conf[:-1, :-1], axis=1).astype(float)
            acc_valid = pos_gt > 0
            acc[acc_valid] = tp[acc_valid] / pos_gt[acc_valid]
            union = pos_gt + pos_pred - tp
            iou_valid = np.logical_and(acc_valid, union > 0)
            iou[iou_valid] = tp[iou_valid] / union[iou_valid]
            macc = np.sum(acc[acc_valid]) / np.sum(acc_valid)
            miou = np.sum(iou[iou_valid]) / np.sum(iou_valid)
            fiou = np.sum(iou[iou_valid] * class_weights[iou_valid])
            pacc = np.sum(tp) / np.sum(pos_gt)
        res = {"mIoU": 100 * miou, "fwIoU": 100 * fiou}
        for i, name in enumerate(self.class_names):
            res[f"IoU-{name}"] = 100 * iou[i]
        res["mACC"] = 100 * macc
        res["pACC"] = 100 * pacc
        for i, name in enumerate(self.class_names):
            res[f"ACC-{name}"] = 100 * acc[i]
        return {"sem_seg": {k: (float(v) if np.isfinite(v) else None) for k, v in res.items()}}


class SyntheticDetectionDataset:
    """BASELINE configs[4] data: COCO-shape synthetic entries (SURVEY §8d.5): uint8 images, 1..20 boxes per image, uniform cxcy in [0.2,0.8], wh in [0.05,0.35]."""

    def __init__(self, n: int = 64, size: int = 640, num_classes: int = 80, seed: int = 4):
        self.n, self.size, self.num_classes, self.seed = n, size, num_classes, seed

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 100003 + i)
        k = int(torch.randint(1, 21, (1,), generator=g))
        c = 0.2 + 0.6 * torch.rand((k, 2), generator=g)
        wh = 0.05 + 0.30 * torch.rand((k, 2), generator=g)
        box = torch.cat([c - wh / 2, c + wh / 2], 1) * self.size
        img = torch.randint(0, 256, (3, self.size, self.size), generator=g, dtype=torch.uint8)
        return {"image": img, "height": self.size, "width": self.size,
                "instances": Instances((self.size, self.size), boxes=Boxes(box), classes=torch.randint(0, self.num_classes, (k,), generator=g))}


class SyntheticSemSegDataset:
    """ADE20K-shaped synthetic semantic-segmentation entries: seeded uint8 images [3,H,W] and label maps `sem_seg` [H,W] uint8 made of class blocks on an
    8x8 grid with about 5% of the pixels set to ignore_label.  The entries take the `sizes` in turn, in consecutive runs (default: two non-square sizes that
    are not multiples of 32).  `metadata.ignore_label` is what inference_on_dataset hands to SemSegEvaluator."""

    def __init__(self, n: int = 8, sizes=((357, 483), (250, 333)), num_classes: int = 150, ignore_label: int = 255, seed: int = 7):
        from types import SimpleNamespace
        self.n, self.sizes, self.num_classes, self.seed = n, [tuple(s) for s in sizes], num_classes, seed
        self.metadata = SimpleNamespace(ignore_label=ignore_label)

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 100003 + i)
        H, W = self.sizes[i * len(self.sizes) // self.n]
        img = torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8)
        blocks = torch.randint(0, self.num_classes, (8, 8), generator=g, dtype=torch.uint8)
        gt = blocks[(torch.arange(H) * 8 // H)[:, None], (torch.arange(W) * 8 // W)[None, :]]
        gt[torch.rand((H, W), generator=g) < 0.05] = self.metadata.ignore_label
        return {"image": img, "height": H, "width": W, "sem_seg": gt}
