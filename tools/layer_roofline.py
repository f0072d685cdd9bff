"""Per-launch timing of one forward (eager, CUDA events around every C-ABI call) with a per-layer roofline estimate.
Run on the GPU:  python tools/layer_roofline.py > layer_roofline.txt"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bench import seeded_weights, measured_peaks
from focoos_b200 import DETRConfig, FAIDetr, ops

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
PREC = sys.argv[2] if len(sys.argv) > 2 else "fp32_tc"   # fp32_tc: the tensor roof of a layer is a THIRD of the fp16 peak (three products per algorithmic product)
pk = measured_peaks()
TENSOR = pk["tf_sustained"] * 1e12 / (3.0 if PREC == "fp32_tc" else 1.0)
m = FAIDetr(DETRConfig(), precision=PREC); m.load_state_dict(seeded_weights(), strict=True); m.cuda()
x = torch.rand(B, 3, 640, 640, device="cuda") * 255
for _ in range(3): m(x)
torch.cuda.synchronize()
tr = ops.enable_trace(True)
m(x)
torch.cuda.synchronize()
ops.enable_trace(False)
rows = []
for name, note, e0, e1 in tr:
    us = e0.elapsed_time(e1) * 1e3
    d = {"sym": name.replace("fb200_", ""), "us": us}
    if isinstance(note, dict) and note.get("op") == "conv":
        n = note; s = n["stride"]; Ho, Wo = (n["H"] + s - 1) // s if n["k"] > 1 else n["H"] // s if s > 1 else n["H"], (n["W"] + s - 1) // s if n["k"] > 1 else n["W"]
        Ho = (n["H"] - 1) // s + 1; Wo = (n["W"] - 1) // s + 1
        M = n["B"] * Ho * Wo; K = n["k"] * n["k"] * n["Cin"]
        flops = 2.0 * M * n["Cout"] * K
        if n.get("algo") == 3 and n["xdt"] == "float16":   # split operands passed as the dense [hi|lo] tensor: Cin counts both planes
            n = dict(n, Cin=n["Cin"] // 2, xdt="pair")
            K = n["k"] * n["k"] * n["Cin"]; flops = 2.0 * M * n["Cout"] * K
        ie = 2 if n["xdt"] == "float16" else 4; oe = 2 if n["odt"] == "float16" else 4   # pair and fp32: 4 bytes per element
        byts = n["B"] * n["H"] * n["W"] * n["Cin"] * ie + n["Cout"] * K * ie + M * n["Cout"] * oe * (2 if n["res"] else 1)
        ideal = max(flops / TENSOR, byts / (pk["hbm_gbs"] * 1e9)) * 1e6
        d.update(desc=f'{n["H"]}x{n["W"]} {n["Cin"]}->{n["Cout"]} k{n["k"]} s{s}{" +res" if n["res"] else ""} {n["odt"][5:]}', gflop=flops / 1e9, mb=byts / 1e6, ideal_us=ideal,
                 tfs=flops / us / 1e6, gbs=byts / us / 1e3, bound="T" if flops / TENSOR > byts / (pk["hbm_gbs"] * 1e9) else "M")
    rows.append(d)
tot = sum(r["us"] for r in rows)
ideal_tot = sum(r.get("ideal_us", 0) for r in rows)
print(f"precision {PREC}: tensor roof per layer = {TENSOR/1e12:.0f} TFLOP/s algorithmic (sustained bf16 peak{' / 3' if PREC == 'fp32_tc' else ''}), HBM {pk['hbm_gbs']:.0f} GB/s")
print(f"B={B}: {len(rows)} launches, sum of per-launch times {tot/1e3:.2f} ms; conv/linear ideal (sum of max(tensor,HBM)) {ideal_tot/1e3:.2f} ms")
print(f"{'#':>3} {'sym':18} {'us':>8} {'ideal':>7} {'eff':>5} {'TF/s':>6} {'GB/s':>6} b  desc")
for i, r in enumerate(rows):
    if "desc" in r:
        print(f"{i:3d} {r['sym']:18} {r['us']:8.1f} {r['ideal_us']:7.1f} {r['ideal_us']/r['us']:5.2f} {r['tfs']:6.0f} {r['gbs']:6.0f} {r['bound']}  {r['desc']}")
    else:
        print(f"{i:3d} {r['sym']:18} {r['us']:8.1f}")
conv = [r for r in rows if "desc" in r]
print("conv/linear total us", round(sum(r["us"] for r in conv), 1), "of", round(tot, 1))
