"""Config 3 of BASELINE.json: fai-mf-l-coco-ins, bs=16, 800x800 on one GPU — images/s of FAIMaskFormer.forward (+ GPU part of the
instance post-process), CUDA events, plus a per-kernel-symbol time breakdown of one eager forward.
    python tools/bench_mf.py [batch] [size]
FB200_BENCH_MODEL picks another fai_mf registry entry (default fai-mf-l-coco-ins; fai-mf-m-coco-ins, fai-mf-s-coco-ins, and the semantic fai-mf-l-ade,
fai-mf-m-ade, whose step ends in the semantic argmax instead of the instance statistics), FB200_BENCH_PRECISION the precision
(default fp16, which also runs fp32_tc in a second process).  FB200_BENCH_LATENCY=N adds the p50 / p90 of N single-image FocoosModel calls (uint8 image at
[size]x[size], CUDA graph replay, post-processing included).  The JSON line carries the card, its power limit, and the median SM clock and the throttle
reasons sampled with nvidia-smi during the timed window."""
import json, os, sys, collections, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from focoos_b200 import ModelManager, ops
from focoos_b200.utils.seeded_weights import seeded_state_dict
from tools.smi import SmiSampler

B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
S = int(sys.argv[2]) if len(sys.argv) > 2 else 800
NAME = os.environ.get("FB200_BENCH_MODEL", "fai-mf-l-coco-ins")
with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", NAME.replace("-", "_") + "_state_dict_manifest.json")) as f:
    man = json.load(f)
sd = seeded_state_dict({k: torch.empty(v[0], dtype=getattr(torch, v[1])) for k, v in man.items()}, 0)
PREC = os.environ.get("FB200_BENCH_PRECISION", "fp16")
fm = ModelManager.get(NAME, state_dict=sd, precision=PREC)
m = fm.model; m.cuda()


x = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, device="cuda")
SEMANTIC = m.config.postprocessing_type == "semantic"
def step_unfused():  # the reference's split: model.forward returns [B,Q,H,W] probabilities, the processor reads them back
    out = m(x)
    return ops.mask_argmax(out.masks, out.logits.max(-1).values) if SEMANTIC else ops.mask_stats(out.masks, 0.5)
def step():          # what FocoosModel.__call__ runs: statistics (instance) or the argmax (semantic) fused into the upsampling (fai_mf.LazyMasks)
    m.lazy_masks = True
    out = m(x)
    m.lazy_masks = False
    lm = out.masks
    if SEMANTIC:
        return ops.mask_sigmoid_upsample_argmax(lm.logits, lm.num_queries, lm.size, out.logits.max(-1).values)
    return ops.mask_sigmoid_upsample_stats(lm.logits, lm.num_queries, lm.size, 0.5)
def timed(fn, n=5):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
ms_unfused = timed(step_unfused)
with SmiSampler() as smi:
    ms = timed(step, int(os.environ.get("FB200_BENCH_STEPS", "5")))
extra = {"gpu": smi.summary()}
LAT = int(os.environ.get("FB200_BENCH_LATENCY", "0"))
if LAT:  # bs=1 through the public path: preprocess, graph replay, post-processing to host detections
    img = torch.randint(0, 256, (S, S, 3), dtype=torch.uint8).numpy()
    for _ in range(5): fm.infer(img, threshold=0.5)
    lat = []
    with SmiSampler() as smi1:
        for _ in range(LAT):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            fm.infer(img, threshold=0.5)
            torch.cuda.synchronize(); lat.append((time.perf_counter() - t0) * 1e3)
    lat.sort()
    extra["bs1_latency_ms"] = {"p50": lat[len(lat) // 2], "p90": lat[int(len(lat) * 0.9)], "n": LAT, "size": S, "gpu": smi1.summary()}
tr = ops.enable_trace(True); step(); torch.cuda.synchronize(); ops.enable_trace(False)
agg = collections.defaultdict(lambda: [0, 0.0])
for name, note, a, b in tr:
    agg[name][0] += 1; agg[name][1] += a.elapsed_time(b)
tot = sum(v[1] for v in agg.values())
print(json.dumps({"workload": f"{NAME} bs={B} {S}x{S}" + (" (BASELINE configs[2])" if NAME == "fai-mf-l-coco-ins" else ""), "images_per_s": B / ms * 1e3, "ms_per_step": ms, "unfused_images_per_s": B / ms_unfused * 1e3, "unfused_ms_per_step": ms_unfused, "dtype": {"fp16": "f16", "fp32_tc": "f32 (3x f16 wgmma products)", "fp32": "f32 SIMT"}[PREC], "precision": PREC, "launches": len(tr),
                  "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9, **extra}))
for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{t:9.2f} ms {100*t/tot:5.1f}%  n={c:4d}  {k}")
if PREC == "fp16" and os.environ.get("FB200_BENCH_PARITY_MODE", "1") == "1":  # the parity-green mode (fp32_tc) of the same workload, in its own process
    import subprocess
    del m, fm, x
    torch.cuda.empty_cache()
    r = subprocess.run([sys.executable] + sys.argv, env=dict(os.environ, FB200_BENCH_PRECISION="fp32_tc", FB200_BENCH_PARITY_MODE="0"), capture_output=True, text=True, timeout=280)
    line = next((l for l in r.stdout.splitlines() if l.startswith("{")), None)
    print("PARITY_MODE " + (line or json.dumps({"error": r.stderr[-300:]})))
