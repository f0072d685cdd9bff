"""Where the time of box-AP model.eval goes: BoxAPEvaluator (matching in Python on the host) against DeviceBoxAPEvaluator (matching kernel + numpy
accumulation), at one GPU and, when the machine has more, at N GPUs.
    python tools/bench_eval.py [images] [repeats]
fai-detr-l-obj365 (fp32_tc) on SyntheticDetectionDataset at 640x640, bs=32, top_k=300, `images` (default 1024) images decoded once before timing.
Per evaluator and repeat (after one warm-up pass): seconds in forward + eval_postprocess, in `process` and in `evaluate`, each window closed by a device
synchronise.  Multi-GPU: wall seconds of FocoosModel.eval(num_gpus=N) against num_gpus=1 on the same (lazily decoded) dataset, process start-up included.
One JSON line per configuration with the median and the min-max spread over the repeats, the card, its power limit and the SM clock during the windows."""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from focoos_b200 import ModelManager  # noqa: E402
from focoos_b200.trainer import BoxAPEvaluator, DeviceBoxAPEvaluator, SyntheticDetectionDataset, TrainerArgs  # noqa: E402
from tools.smi import SmiSampler  # noqa: E402

IMAGES = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
REPEATS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
BS, SIZE, TOP_K, NAME = 32, 640, 300, "fai-detr-l-obj365"


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        return None


@torch.no_grad()
def phases(fm, data, evaluator):
    """(forward + eval_postprocess, process, evaluate) seconds of one pass of inference_on_dataset's loop, and the metrics"""
    t = [0.0, 0.0, 0.0]
    evaluator.reset()
    for s in range(0, len(data), BS):
        entries = data[s:s + BS]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fm.model(torch.stack([e["image"] for e in entries]).cuda().float())
        pp = fm.processor.eval_postprocess(out, entries, TOP_K)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        evaluator.process(entries, pp)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        t[0] += t1 - t0
        t[1] += t2 - t1
    t0 = time.perf_counter()
    metrics = evaluator.evaluate()
    torch.cuda.synchronize()
    t[2] = time.perf_counter() - t0
    return t, metrics


def summary(samples):
    return {"median": round(statistics.median(samples), 4), "min": round(min(samples), 4), "max": round(max(samples), 4)}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a GPU; none is visible")
    fm = ModelManager.get(NAME, precision="fp32_tc")
    lazy = SyntheticDetectionDataset(n=IMAGES, size=SIZE, num_classes=365)
    data = [lazy[i] for i in range(IMAGES)]
    common = {"model": NAME, "precision": "fp32_tc", "size": f"{SIZE}x{SIZE}", "bs": BS, "top_k": TOP_K, "images": IMAGES, "repeats": REPEATS,
              "power_limit": power_limit()}
    results = {}
    for label, cls in (("BoxAPEvaluator", BoxAPEvaluator), ("DeviceBoxAPEvaluator", DeviceBoxAPEvaluator)):
        ev = cls(365)
        phases(fm, data[: 2 * BS], ev)  # warm-up: engine, kernels, allocator
        runs = []
        with SmiSampler() as smi:
            for _ in range(REPEATS):
                runs.append(phases(fm, data, ev))
        results[label] = runs[0][1]
        t = list(zip(*[r[0] for r in runs]))
        print(json.dumps({**common, "evaluator": label, "forward_postprocess_s": summary(t[0]), "process_s": summary(t[1]), "evaluate_s": summary(t[2]),
                          "total_s": summary([sum(r[0]) for r in runs]), "gpu": smi.summary()}), flush=True)
    print(json.dumps({**common, "same_metrics": results["BoxAPEvaluator"] == results["DeviceBoxAPEvaluator"], "metrics": results["DeviceBoxAPEvaluator"]}),
          flush=True)
    n = torch.cuda.device_count()
    if n > 1:
        for gpus in (1, n):
            walls, got = [], None
            for r in range(REPEATS):
                with tempfile.TemporaryDirectory() as tmp:
                    args = TrainerArgs(run_name="e", output_dir=tmp, batch_size=BS, num_gpus=gpus, master_port=29571 + r)
                    t0 = time.perf_counter()
                    got = fm.eval(args, lazy, save_json=False)
                    walls.append(time.perf_counter() - t0)
            print(json.dumps({**common, "num_gpus": gpus, "model_eval_wall_s": summary(walls), "metrics": got}), flush=True)
    else:
        print(json.dumps({**common, "num_gpus": n, "multi_gpu": "not measured: one GPU visible"}), flush=True)


if __name__ == "__main__":
    main()
