"""fai-detr-m-coco (STDC-2 trunk, 3 decoder layers, 80 classes) inference throughput and latency on one GPU.

    python tools/bench_detr_m.py [--batch 32] [--steps 20] [--warmup 5] [--precisions fp16,fp32_tc]

Each precision runs in its own process (seeded weights, synthetic 640x640 uint8 images resident in HBM) and prints one JSON line:
  * images/s at bs=--batch: CUDA-graph replay of FAIDetr.forward + the fused DETR post-process (ops.detr_postprocess), CUDA events around --steps steps;
  * bs=1 p50 / p90 latency of forward + post-process through FocoosModel's CUDA-graph cache (FocoosModel._forward replays the captured graph),
    device-timed per iteration;
  * per-kernel totals of one bs=--batch forward from ops.enable_trace (a separate, traced pass: tracing is off while timing);
  * the card name and power limit, and the median SM clock sampled during the timed window of the same run."""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

NAME = "fai-detr-m-coco"


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def run(precision, B, steps, warmup):
    from bench import ClockSampler, _graphed, _latency
    from focoos_b200 import DETRConfig, FAIDetr, FocoosModel, ModelInfo, ops
    from focoos_b200.model_manager import _REGISTRY
    from oracle.gen_golden import synth_images
    from tests.parity_utils import seeded_sd

    dev = torch.device("cuda", 0)
    m = FAIDetr(DETRConfig.from_dict(_REGISTRY[NAME]["config"]), precision=precision)
    m.load_state_dict(seeded_sd(0, "fai_detr_m_coco"), strict=True)
    fm = FocoosModel(m, ModelInfo(name=NAME, im_size=640))
    fm.model.to(dev)
    x = torch.from_numpy(np.stack(synth_images(1, [(640, 640)] * B))).to(dev)
    sizes = torch.tensor([(640, 640)] * B, dtype=torch.int32, device=dev)

    def step():
        o = fm.model(x)
        return ops.detr_postprocess(o.logits, o.boxes, sizes, 300, 0.5)

    replay = _graphed(step, True)
    for _ in range(warmup):
        replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(0) as clk:
        e0.record()
        for _ in range(steps):
            replay()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps

    x1, s1 = x[:1].contiguous(), sizes[:1].contiguous()

    def step1():  # FocoosModel's graph cache: first sighting eager, second captures, then replays
        o = fm._forward(x1)
        return ops.detr_postprocess(o.logits, o.boxes, s1, 300, 0.5)

    lat = _latency(step1, False)
    assert len(fm._graphs) == 1, "bs=1 latency did not run through the CUDA-graph cache"

    tr = ops.enable_trace(True)
    fm.model(x)
    torch.cuda.synchronize()
    ops.enable_trace(False)
    agg = collections.defaultdict(lambda: [0, 0.0])
    for name, _, a, b in tr:
        agg[name][0] += 1
        agg[name][1] += a.elapsed_time(b)
    kernels = [{"kernel": k, "launches": c, "ms": round(t, 3)} for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])]
    return {"model": NAME, "precision": precision, "batch": B, "images_per_s": round(B / ms * 1e3, 1), "ms_per_step": round(ms, 3), "steps": steps,
            "bs1_p50_ms": round(lat["p50_ms"], 3), "bs1_p90_ms": round(lat["p90_ms"], 3), "launches_per_forward": len(tr), "kernels": kernels,
            "card": card(), "clocks": clk.summary(), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precisions", default="fp16,fp32_tc")
    ap.add_argument("--one", default=None, help=argparse.SUPPRESS)  # child process: run this precision only
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_detr_m needs a GPU"
    if args.one:
        print(json.dumps(run(args.one, args.batch, args.steps, args.warmup)))
        return
    for p in args.precisions.split(","):  # one process per precision: neither run sees the other's allocator state or packed weights
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", p, "--batch", str(args.batch), "--steps", str(args.steps),
                            "--warmup", str(args.warmup)], capture_output=True, text=True, timeout=900)
        line = next((ln for ln in r.stdout.splitlines() if ln.startswith("{")), None)
        print(line or json.dumps({"precision": p, "error": r.stderr[-800:]}), flush=True)


if __name__ == "__main__":
    main()
