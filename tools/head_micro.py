"""In-graph timing of the two halves of the fp32_tc DETR forward (trunk = backbone + hybrid encoder + decoder input projection; head = value / enc_output
projections + query selection + 6 decoder layers + score head), each captured in its own CUDA graph.
    python tools/head_micro.py          # trunk / head split
    python tools/head_micro.py attn     # the split-precision attention kernel alone (decoder 300x300 and AIFI 400x400 shapes)
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import seeded_weights
from focoos_b200 import DETRConfig, ops
from focoos_b200.fai_detr import FAIDetr

dev = torch.device("cuda", 0)


def time_graph(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


if "attn" in sys.argv:
    for B, L in ((32, 300), (32, 400)):
        qk = torch.randn((B, L, 512), device=dev)
        v = torch.randn((B, L, 256), device=dev)
        f = lambda: ops.attention(qk[..., :256], qk[..., 256:], v, 8, 1.0 / math.sqrt(32), split=True, out_pair=True)
        print(f"attention_split B={B} L={L}: {time_graph(f, 50) * 1e3:8.1f} us")
    sys.exit(0)

B = 32
model = FAIDetr(DETRConfig(), precision="fp32_tc")
model.load_state_dict(seeded_weights(), strict=True)
model.to(dev)
eng = model.engine()
x = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (B, 640, 640, 3), dtype=np.uint8)).to(dev)

with torch.no_grad():
    state = {}

    def trunk():
        state["mem"], state["shapes"], state["K"] = eng._trunk(x, None)

    def head():
        mem, shapes, K = state["mem"], state["shapes"], state["K"]
        value_all = eng._linear(eng.value_all, mem)
        t = eng._linear(eng.enc_output, mem)
        return eng._forward_head(t, value_all, mem, shapes, K, B, mem.shape[1], None)

    l0 = ops.launch_count()
    trunk()
    l1 = ops.launch_count()
    head()
    l2 = ops.launch_count()
    t_tr = time_graph(trunk)
    t_hd = time_graph(head)
    t_all = time_graph(lambda: model(x))
    print(f"trunk {t_tr:7.3f} ms ({l1 - l0} launches)  head {t_hd:7.3f} ms ({l2 - l1} launches)  whole forward {t_all:7.3f} ms")
