"""`FocoosModel.train` / `FocoosModel.eval` for the fai-detr family — the slice of the reference's trainer that sits ON the hot path
(SURVEY §3.3/§3.5, §8 a21/f3):

  TrainerLoop.run_step              focoos/trainer/trainer.py:723-773      -> train_step.TrainStep (forward, criterion, backward, exchange, AdamW)
  DETRProcessor.preprocess (train)  focoos/models/fai_detr/processor.py:66-100 -> `training_batch` below (DatasetEntry list -> images + DETRTargets)
  WarmupMultiStepLR                 focoos/trainer/solver/lr_scheduler.py:73-110 -> `lr_factor`
  run_train / launch                focoos/trainer/trainer.py:283-420, utils/distributed/dist.py:40-137 -> `run_train_entry` (one process per GPU, NCCL)
  inference_on_dataset              focoos/trainer/evaluation/evaluator.py:115-238 -> `inference_on_dataset` (batched, instances stay on the device)

Out of scope (reference control plane, SURVEY §2): hooks, checkpointer rotation, EMA, Hub sync, tensorboard, COCO-json evaluators (pycocotools);
`BoxAPEvaluator` below is a small self-contained AP@[.5:.95] / AP50 so that `model.eval` returns numbers without those dependencies.

Dataset contract (reference `MapDataset` of `DatasetEntry`, ports.py): `len(ds)`, `ds[i]` -> entry with `.image` (uint8 / float tensor [3,H,W]),
`.height`, `.width`, `.instances` with `.boxes.tensor` ([n,4] absolute xyxy in the image's pixels) and `.classes` ([n] int64); plain dicts with the
same keys are accepted.  Images of one batch must share one size that is a multiple of 32 (the reference pads with ImageList; the synthetic
COCO-shape data of BASELINE configs[4] is 640x640).
"""
from __future__ import annotations

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
    from .train_step import FlatAdamW, GradBucketReducer, TrainStep, get_optimizer_params
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
    step = TrainStep(model, opt, red)
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
    metrics = None
    if data_val is not None and rank == 0:
        model.eval()
        metrics = inference_on_dataset(fm, data_val, batch_size=args.batch_size)
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


@torch.no_grad()
def inference_on_dataset(fm, dataset, batch_size: int = 16, evaluator: Optional[BoxAPEvaluator] = None, top_k: Optional[int] = None):
    """evaluator.py:115-238: run the model over `dataset` in batches (the reference uses batch 1 per GPU), `processor.eval_postprocess`, `evaluator.process`;
    each rank takes a contiguous shard and rank 0 evaluates its own (single-process evaluation is the tested path)."""
    model, proc = fm.model, fm.processor
    model.eval()
    evaluator = evaluator or BoxAPEvaluator(model.config.num_classes)
    evaluator.reset()
    lo, hi = D.shard_range(len(dataset))
    for s in range(lo, hi, batch_size):
        entries = [dataset[i] for i in range(s, min(hi, s + batch_size))]
        x = torch.stack([torch.as_tensor(_get(e, "image")) for e in entries]).to(model.device).float()
        out = model(x)
        evaluator.process(entries, proc.eval_postprocess(out, entries, top_k))
    return evaluator.evaluate()


def run_eval_entry(fm, args: TrainerArgs, data_test, save_json: bool = True):
    assert args.num_gpus, "Testing without GPUs is not supported. num_gpus must be greater than 0"  # focoos_model.py:300
    metrics = inference_on_dataset(fm, data_test, batch_size=args.batch_size)
    fm.model_info.val_metrics = metrics
    if save_json:
        out_dir = os.path.join(args.output_dir, args.run_name)
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "eval_metrics.json"), "w") as f:
            json.dump(metrics, f, indent=1)
    return metrics


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
