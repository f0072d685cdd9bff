"""Images/s of semantic model.eval (inference_on_dataset with SemSegEvaluator) beside the torch formulation of the reference's evaluation tail.
    python tools/bench_sem_seg_eval.py [batches]
For fai-mf-m-ade and bisenetformer-m-ade (seeded weights, precision fp32_tc and fp16) on SyntheticSemSegDataset at 640x640, bs=16, `batches` (default 8)
timed batches after one warm-up pass over the same data:
  * "focoos_b200": inference_on_dataset, i.e. the model with lazy masks, eval_postprocess (NHWC probabilities + per-image 1x1 product) and the confusion kernel;
  * "torch_tail": the same model returning the materialised [B,Q,H,W] probabilities, then per image the reference's torch.einsum("qc,qhw->chw"),
    argmax(0) and bincount on the GPU, the matrix kept on the device.
One JSON line per (model, precision), with the card, its power limit and the SM clock / throttle reasons sampled during each timed window."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from focoos_b200 import ModelManager  # noqa: E402
from focoos_b200.trainer import SyntheticSemSegDataset, inference_on_dataset  # noqa: E402
from focoos_b200.utils.seeded_weights import seeded_state_dict  # noqa: E402
from tools.smi import SmiSampler  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCHES = int(sys.argv[1]) if len(sys.argv) > 1 else 8
BS, SIZE = 16, (640, 640)


def torch_tail(fm, data):
    model = fm.model
    C = model.config.num_classes
    conf = torch.zeros(((C + 1) ** 2,), dtype=torch.int64, device="cuda")
    for s in range(0, len(data), BS):
        entries = [data[i] for i in range(s, min(len(data), s + BS))]
        out = model(torch.stack([e["image"] for e in entries]).cuda().float())
        for i, e in enumerate(entries):
            pred = torch.einsum("qc,qhw->chw", out.logits[i], out.masks[i]).argmax(0)
            gt = e["sem_seg"].cuda().long()
            gt[gt == 255] = C
            conf += torch.bincount((C + 1) * pred.reshape(-1) + gt.reshape(-1), minlength=(C + 1) ** 2)
    return conf


def timed(fn):
    fn()  # warm-up over the same shapes
    torch.cuda.synchronize()
    with SmiSampler() as smi:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    return round(BATCHES * BS / dt, 1), smi.summary()


for name in ("fai-mf-m-ade", "bisenetformer-m-ade"):
    with open(os.path.join(ROOT, "tests", "golden", name.replace("-", "_") + "_state_dict_manifest.json")) as f:
        man = json.load(f)
    sd = seeded_state_dict({k: torch.empty(v[0], dtype=getattr(torch, v[1])) for k, v in man.items()}, 0)
    data = SyntheticSemSegDataset(n=BATCHES * BS, sizes=(SIZE,))
    data = [data[i] for i in range(len(data))]  # decoded once: the timed windows hold the device work and its host feed only
    for precision in ("fp32_tc", "fp16"):
        fm = ModelManager.get(name, state_dict=sd, precision=precision)
        ours, smi_ours = timed(lambda: inference_on_dataset(fm, data, batch_size=BS))
        with torch.no_grad():
            ref, smi_ref = timed(lambda: torch_tail(fm, data))
        print(json.dumps({"model": name, "precision": precision, "size": f"{SIZE[0]}x{SIZE[1]}", "bs": BS, "images": BATCHES * BS,
                          "focoos_b200_img_s": ours, "torch_tail_img_s": ref, "gpu_focoos_b200": smi_ours, "gpu_torch_tail": smi_ref}), flush=True)
        del fm
        torch.cuda.empty_cache()
