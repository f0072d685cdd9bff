"""BASELINE.json configs[4]: fai-detr-l fine-tune, bs=16/GPU, 640x640, synthetic COCO-shape targets (80 classes, 1..20 boxes per image),
data-parallel gradient all-reduce over NCCL.  One "step" = TrainerLoop.run_step: training forward, criterion, backward, gradient
exchange, clip x2 + AdamW with loss scaling.

    python tools/bench_train.py [--batch 16] [--steps 5] [--warmup 2] [--precision fp32_tc]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29512 tools/bench_train.py

Prints one JSON line (images/s over all ranks, device-timed, max over ranks) plus a per-phase breakdown of one step."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from focoos_b200 import DETRConfig, FAIDetr, ops  # noqa: E402
from focoos_b200 import distributed as D  # noqa: E402
from focoos_b200.criterion import DETRTargets  # noqa: E402
from focoos_b200.train_step import FlatAdamW, GradBucketReducer, ModelEMA, TrainStep, get_optimizer_params  # noqa: E402
from focoos_b200.utils.seeded_weights import desaturate_classifiers, seeded_state_dict  # noqa: E402


def run_leg(batch=16, size=640, steps=5, warmup=2, precision="fp32_tc", by_symbol=True, sync_bn=None, ema=False):
    """One fine-tune leg on the ALREADY-INITIALISED process group (every rank calls it); returns the result dict on every rank.  ema: with the model EMA
    (TrainerArgs.ema_enabled defaults: decay 0.999, warmup 2000) updated after every step."""
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = torch.device("cuda", local)
    cfg = DETRConfig(num_classes=80)
    m = FAIDetr(cfg, precision="fp32_tc" if precision == "amp" else precision)
    m.train_precision = precision
    m.load_state_dict(desaturate_classifiers(seeded_state_dict(m.state_dict(), seed=0)), strict=True)  # same parameters on every rank
    m.to(dev).train()
    if sync_bn is not None and hasattr(m, "sync_bn"):
        m.sync_bn = bool(sync_bn)
    opt = FlatAdamW(get_optimizer_params(m, base_lr=5e-4, weight_decay=0.02, weight_decay_norm=0.0, backbone_multiplier=0.1), clip_gradients=0.1, amp=True, world_size=world)
    opt.track_unused_parameters()
    red = GradBucketReducer(opt)
    red.attach_hooks()
    step = TrainStep(m, opt, red, ModelEMA(m, opt) if ema else None)
    g = torch.Generator().manual_seed(4 + rank)  # SURVEY 8(d).5: seed 4 + rank
    x = torch.randint(0, 256, (batch, 3, size, size), generator=g).float().to(dev)
    targets = []
    for _ in range(batch):
        n = int(torch.randint(1, 21, (1,), generator=g))
        box = torch.cat([0.2 + 0.6 * torch.rand((n, 2), generator=g), 0.05 + 0.30 * torch.rand((n, 2), generator=g)], 1)
        targets.append(DETRTargets(labels=torch.randint(0, 80, (n,), generator=g).to(dev), boxes=box.to(dev)))
    for _ in range(warmup):
        step(x, targets)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    l0 = ops.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.reset_peak_memory_stats()
    e0.record()
    for _ in range(steps):
        losses = step(x, targets)
    e1.record()
    torch.cuda.synchronize()
    ms = D.max_over_ranks(e0.elapsed_time(e1) / steps, dev)
    launches = (ops.launch_count() - l0) // steps
    # one more step, phase by phase
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    opt.zero_grad()
    ev[0].record()
    loss_dict = m(x, targets).loss
    ev[1].record()
    opt.scale_loss(sum(loss_dict.values())).backward()
    ev[2].record()
    red.finish()
    ev[3].record()
    opt.step()
    ev[4].record()
    torch.cuda.synchronize()
    phases = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(["forward_and_criterion_ms", "backward_ms", "exchange_tail_ms", "optimizer_ms"])}
    # per-symbol device time of one more step (CUDA events around every C-ABI call; torch glue = the remainder)
    by_sym = {}
    if by_symbol and os.environ.get("FB200_TRACE", "1") == "1":
        tr = ops.enable_trace(True)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        step(x, targets)
        t1.record()
        torch.cuda.synchronize()
        for name, _, a, b_ in tr:
            d = by_sym.setdefault(name.replace("fb200_", ""), [0, 0.0])
            d[0] += 1
            d[1] += a.elapsed_time(b_)
        ops.enable_trace(False)
        by_sym = {k: {"n": v[0], "ms": round(v[1], 3)} for k, v in sorted(by_sym.items(), key=lambda kv: -kv[1][1])}
        by_sym["_step_total_ms"] = t0.elapsed_time(t1)
        by_sym["_kernels_ms"] = round(sum(v["ms"] for k, v in by_sym.items() if isinstance(v, dict)), 3)
    total = float(sum(v.detach() for v in losses.values()))
    res = {"metric": "images/sec fai-detr-l fine-tune step (fwd + criterion + bwd + all-reduce + AdamW)", "value": batch * world / (ms / 1e3), "unit": "images/s",
           "n_gpus": world, "ms_per_step": ms, "steps": steps, "warmup": warmup, "scaling": "weak", "dtype": "f32 storage; " + {"fp32_tc": "3x f16 wgmma products for conv/linear forward, data and weight gradients", "fp32": "SIMT f32",
                                                                      "amp": "ONE f16 wgmma product (fp16-rounded operands, f32 accumulation) for conv/linear forward, data and weight gradients - the reference's torch.autocast(fp16) + GradScaler arithmetic (trainer/trainer.py:735)"}[precision],
           "precision": precision,
           "config": {"workload": f"fai-detr-l (80 classes) bs={batch}/GPU {size}x{size} synthetic COCO-shape targets (BASELINE configs[4])", "global_batch": batch * world,
                      "sync_bn": bool(getattr(m, "sync_bn", False)) and world > 1, "ema": bool(ema)},
           "kernel_launches_per_step": launches, "phases_ms": phases, "peak_mem_GB": torch.cuda.max_memory_allocated() / 1e9, "loss_total": total, "optimizer": opt.stats(), "by_symbol": by_sym}
    red.detach_hooks() if hasattr(red, "detach_hooks") else None
    del step, red, opt, m, x, targets
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--precision", default="fp32_tc", choices=["fp32", "fp32_tc", "amp"])
    ap.add_argument("--no-sync-bn", action="store_true")
    ap.add_argument("--ema", action="store_true")
    args = ap.parse_args()
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(local)
    D.init_from_env("nccl", torch.device("cuda", local))
    res = run_leg(args.batch, args.size, args.steps, args.warmup, args.precision, sync_bn=False if args.no_sync_bn else None, ema=args.ema)
    if rank == 0:
        print(json.dumps(res))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
