"""Cost of running the segmentation models at their true image size instead of the next multiple of 32.

    python tools/bench_any_size.py [--steps N] [--warmup W] [--precisions fp32_tc,fp16]

Times FAIMaskFormer at bs=1 and bs=8 on 720x1280 against 736x1280 and BisenetFormer at bs=1 on 1080x1920 against 1088x1920 (CUDA events around
model.forward on a uint8 NHWC batch), and lists the per-launch time of every 3x3 stride-2 conv of one forward: at the odd sizes these read their input
through the strided tensor map, at the even sizes through the parity view.  Prints one JSON line per workload and the GPU it ran on."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from focoos_b200 import ops  # noqa: E402
from focoos_b200.bisenetformer import BisenetFormer, BisenetFormerConfig  # noqa: E402
from focoos_b200.fai_mf import FAIMaskFormer, MaskFormerConfig  # noqa: E402
from focoos_b200.utils.seeded_weights import seeded_state_dict  # noqa: E402
from tests.parity_utils import manifest_template  # noqa: E402

WORKLOADS = [("fai-mf-l-coco-ins", 1, (720, 1280), (736, 1280)), ("fai-mf-l-coco-ins", 8, (720, 1280), (736, 1280)),
             ("bisenetformer-l-ade", 1, (1080, 1920), (1088, 1920))]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def model(name, precision):
    if name.startswith("fai-mf"):
        m, man = FAIMaskFormer(MaskFormerConfig(), precision=precision), "fai_mf_l_coco_ins"
    else:
        m, man = BisenetFormer(BisenetFormerConfig(), precision=precision), "bisenetformer_l_ade"
    m.load_state_dict(seeded_state_dict(manifest_template(man), 0), strict=True)
    m.lazy_masks = True  # what FocoosModel.__call__ runs: the final upsampling is fused into the post-process
    return m.cuda()


def time_forward(m, x, steps, warmup):
    for _ in range(warmup):
        m(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m(x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def s2_convs(m, x, reps=5):
    """per-launch time of each 3x3 stride-2 conv of one forward (median over `reps` traced forwards), keyed by its input map"""
    per = {}
    for _ in range(reps):
        tr = ops.enable_trace(True)
        m(x)
        torch.cuda.synchronize()
        ops.enable_trace(False)
        for i, (name, note, a, b) in enumerate(tr):
            if isinstance(note, dict) and note.get("op") == "conv" and note.get("stride") == 2 and note.get("k") == 3:
                view = "strided" if note["H"] % 2 or note["W"] % 2 else "parity"
                key = (i, f"{note['Cin']}->{note['Cout']} {note['H']}x{note['W']} {note['xdt']}->{note['odt']} {view}")
                per.setdefault(key, []).append(a.elapsed_time(b) * 1e3)
    return [(k[1], sorted(v)[len(v) // 2]) for k, v in sorted(per.items())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precisions", default="fp32_tc,fp16")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_any_size needs a GPU"
    print(json.dumps({"gpu": gpu_info()}))
    for precision in args.precisions.split(","):
        for name, B, odd, even in WORKLOADS:
            m = model(name, precision)
            xs = {s: torch.randint(0, 256, (B, s[0], s[1], 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).cuda() for s in (odd, even)}
            ms = {}
            for rep in range(2):  # alternate the two sizes: drift on a shared machine hits both
                for s in (odd, even):
                    ms.setdefault(s, []).append(time_forward(m, xs[s], args.steps, args.warmup))
            convs = {s: s2_convs(m, xs[s]) for s in (odd, even)}
            pairs = [{"odd": a[0], "odd_us": round(a[1], 1), "even": b[0], "even_us": round(b[1], 1)} for a, b in zip(convs[odd], convs[even])]
            print(json.dumps({"model": name, "precision": precision, "batch": B,
                              f"{odd[0]}x{odd[1]}_ms": round(min(ms[odd]), 3), f"{even[0]}x{even[1]}_ms": round(min(ms[even]), 3),
                              f"{odd[0]}x{odd[1]}_img_s": round(B / min(ms[odd]) * 1e3, 1), f"{even[0]}x{even[1]}_img_s": round(B / min(ms[even]) * 1e3, 1),
                              "stride2_convs": pairs}))
            del m, xs
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
