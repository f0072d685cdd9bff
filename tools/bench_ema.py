"""Cost of the model EMA (TrainerArgs.ema_enabled) on the fai-detr-l fine-tune.

    python tools/bench_ema.py [--launches 200] [--steps 6] [--rounds 2]

1. The EMA launch alone (ops.ema_update, CUDA events over `--launches` launches) on the fai-detr-l-obj365 training state, next to the reference's
   torch._foreach_mul_ + torch._foreach_add_ (plus its per-tensor int64 update) over the same tensors.  Bytes per update, from the shapes: every
   fp32 entry reads the EMA and the weight and writes the EMA (12 B / element), every int64 entry 24 B / element.
2. The step time at bs=16 640x640 in amp precision with and without the EMA (tools/bench_train.run_leg), the two legs alternated `--rounds` times.

Prints one JSON line with the card's name and power limit."""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from focoos_b200 import DETRConfig, FAIDetr, ops  # noqa: E402
from focoos_b200.train_step import FlatAdamW, ModelEMA, get_optimizer_params  # noqa: E402
from focoos_b200.utils.seeded_weights import seeded_state_dict  # noqa: E402
from tools import bench_train  # noqa: E402
from tools.smi import SmiSampler  # noqa: E402


def _time(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def launch_cost(launches):
    dev = torch.device("cuda", 0)
    m = FAIDetr(DETRConfig(num_classes=80), precision="fp32_tc")
    m.load_state_dict(seeded_state_dict(m.state_dict(), seed=0), strict=True)
    m.to(dev).train()
    opt = FlatAdamW(get_optimizer_params(m, 5e-4, 0.02))
    ema = ModelEMA(m, opt)
    ema_ms = _time(ema.update, launches)
    entries = list(m.named_parameters()) + list(m.named_buffers())
    ref = {n: t.detach().clone() for n, t in entries}
    fl = [n for n, t in entries if t.dtype == torch.float32]
    ema_list, vals = [ref[n] for n in fl], [t for n, t in entries if t.dtype == torch.float32]
    others = [(ref[n], t) for n, t in entries if t.dtype != torch.float32]
    d = 0.999 * (1 - math.exp(-1 / 2000))

    def foreach():
        torch._foreach_mul_(ema_list, d)
        torch._foreach_add_(ema_list, vals, alpha=1 - d)
        for e, v in others:
            e.copy_(e * d + v * (1.0 - d))

    def foreach_fp32_only():
        torch._foreach_mul_(ema_list, d)
        torch._foreach_add_(ema_list, vals, alpha=1 - d)

    torch_ms, torch_fp32_ms = _time(foreach, launches), _time(foreach_fp32_only, launches)
    n_fp32 = sum(t.numel() for _, t in entries if t.dtype == torch.float32)
    n_i64 = sum(t.numel() for _, t in entries if t.dtype == torch.int64)
    arena = ema.arena.numel()
    bytes_ = 12 * n_fp32 + 24 * n_i64
    return {"arena_elements": arena, "fp32_elements": n_fp32, "int64_elements": n_i64, "side_chunks": int(ema.chunks.shape[0]), "bytes_per_update": bytes_,
            "ema_update_ms": ema_ms, "ema_update_GBps": bytes_ / ema_ms / 1e6,
            "torch_foreach_ms": torch_ms, "torch_foreach_fp32_only_ms": torch_fp32_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    with SmiSampler() as smi:
        res = {"launch": launch_cost(args.launches)}
        torch.cuda.empty_cache()
        legs = {"off": [], "on": []}
        for _ in range(args.rounds):
            for key, on in (("off", False), ("on", True)):
                r = bench_train.run_leg(batch=16, size=640, steps=args.steps, warmup=2, precision="amp", by_symbol=False, ema=on)
                legs[key].append(r["ms_per_step"])
    res["step_ms"] = legs
    res["step_ms_median"] = {k: sorted(v)[len(v) // 2] for k, v in legs.items()}
    res["gpu"] = smi.summary()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
