"""Single-image latency of the segmentation models through FocoosModel.infer, with the post-processing tail split out.
    python tools/bench_seg_tail.py [calls]
For fai-mf-m-ade, fai-mf-l-ade and bisenetformer-m-ade at 640x640 and fai-mf-l-coco-ins at 1080x1920 (seeded weights, precision fp32_tc, a seeded uint8
image, threshold 0.5 as the README's latency rows): p50 / p90 of `calls` (default 50) infer calls after 5 warm-ups, the median of the preprocess / inference /
postprocess split FocoosDetections.latency carries, the kept-mask count, and - where ops.mask_png exists - the median CUDA-event time of the device PNG
encoder per call.  The tool runs unchanged on trees without the encoder, so two versions can be timed alternately in one session.  One JSON line per model,
with the card, its power limit and the SM clock sampled during the timed calls."""
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from focoos_b200 import ModelManager, ops  # noqa: E402
from focoos_b200.utils.seeded_weights import seeded_state_dict  # noqa: E402
from tools.smi import SmiSampler  # noqa: E402

WORKLOADS = [("fai-mf-m-ade", (640, 640)), ("fai-mf-l-ade", (640, 640)), ("bisenetformer-m-ade", (640, 640)), ("fai-mf-l-coco-ins", (1080, 1920))]
CALLS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

enc_ms = []
if hasattr(ops, "mask_png"):
    _mask_png = ops.mask_png

    def _timed_mask_png(masks, boxes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        data, lengths = _mask_png(masks, boxes)  # returns after reading the lengths, so the end event has completed by the next line
        e1.record()
        e1.synchronize()
        enc_ms.append(e0.elapsed_time(e1))
        return data, lengths

    ops.mask_png = _timed_mask_png

for name, size in WORKLOADS:
    with open(os.path.join(ROOT, "tests", "golden", name.replace("-", "_") + "_state_dict_manifest.json")) as f:
        man = json.load(f)
    sd = seeded_state_dict({k: torch.empty(v[0], dtype=getattr(torch, v[1])) for k, v in man.items()}, 0)
    fm = ModelManager.get(name, state_dict=sd, precision="fp32_tc")
    fm.model.cuda()
    img = torch.randint(0, 256, (*size, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).numpy()
    for _ in range(5):
        fm.infer(img, threshold=0.5)
    lat, split, kept, per_call_enc = [], [], [], []
    with SmiSampler() as smi:
        for _ in range(CALLS):
            n0 = len(enc_ms)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dets = fm.infer(img, threshold=0.5)
            torch.cuda.synchronize()
            lat.append((time.perf_counter() - t0) * 1e3)
            split.append(dets.latency)
            kept.append(len(dets.detections))
            per_call_enc.append(sum(enc_ms[n0:]))
    lat.sort()
    print(json.dumps({"model": name, "size": f"{size[0]}x{size[1]}", "precision": "fp32_tc", "calls": CALLS, "p50_ms": round(lat[len(lat) // 2], 2),
                      "p90_ms": round(lat[int(len(lat) * 0.9)], 2),
                      "split_ms_median": {k: round(statistics.median(s[k] for s in split) * 1e3, 1) for k in ("preprocess", "inference", "postprocess")},
                      "kept_masks": statistics.median(kept), "encoder_ms_median": round(statistics.median(per_call_enc), 3) if hasattr(ops, "mask_png") else None,
                      "gpu": smi.summary()}), flush=True)
    del fm
    torch.cuda.empty_cache()
