#!/usr/bin/env python
"""Per-stage precision budget of the fai-detr-l path on the GPU.

For each precision ("fp16", "fp32", "fp32_tc"; default: all three) this prints, against the reference goldens
(tests/golden/detr_l_obj365_{b2_640,b3_ragged}.npz) and the CPU oracle on a fresh input: backbone / encoder tap errors, encoder query-set overlap,
max |d score| / |d box| on the common queries, and how many thresholded (class, int box) detections are identical.
Output: error_budget.json in the working directory + a table on stdout.  Test/measurement infrastructure (imports oracle/)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from focoos_b200 import DETRConfig, DETRProcessor, FAIDetr  # noqa: E402
from oracle import detr_oracle as O  # noqa: E402
from oracle.gen_golden import synth_images  # noqa: E402
from tests.parity_utils import load_golden, seeded_sd  # noqa: E402


def common_err(g_scores, g_boxes, g_keys, scores, boxes, keys):
    ds = db = 0.0
    for i in range(len(g_keys)):
        pos = {int(k): j for j, k in enumerate(keys[i].tolist())}
        rows = [(j, pos[int(k)]) for j, k in enumerate(g_keys[i].tolist()) if int(k) in pos]
        a, b = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
        ds = max(ds, float(np.abs(g_scores[i][a] - scores[i][b]).max()))
        db = max(db, float(np.abs(g_boxes[i][a] - boxes[i][b]).max()))
    return ds, db


def tap_slice(v, name):
    v = v.permute(0, 3, 1, 2).float().cpu()
    return v[:, :: max(1, v.shape[1] // 8)][:, :8, :: max(1, v.shape[2] // 20), :: max(1, v.shape[3] // 20)].numpy()


def run_case(m, proc, imgs, ref, thr):
    x, _ = proc.preprocess(imgs, device=m.device)
    taps = {}
    out = m(x, taps=taps)
    torch.cuda.synchronize()
    r = {}
    for t in ("res3", "res5", "fpn1", "pan1"):
        if "tap_" + t in ref:
            r[t] = float(np.abs(tap_slice(taps[t], t) - ref["tap_" + t]).max() / ref["tapstat_" + t][2])
    keys = taps["topk_ind"].cpu().numpy()
    r["overlap"] = [len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ref["enc_topk_ind"], keys)]
    r["dscore"], r["dbox"] = common_err(ref["scores"], ref["boxes"], ref["enc_topk_ind"], out.logits.cpu().numpy(), out.boxes.cpu().numpy(), keys)
    dets = proc.postprocess(out, imgs, threshold=thr)
    same = tot = got_n = 0
    for i, d in enumerate(dets):
        n = int(ref["det_count"][i])
        rs = set(zip(ref["det_labels"][i, :n].tolist(), map(tuple, ref["det_boxes"][i, :n].tolist())))
        got = set((x_.cls_id, tuple(x_.bbox)) for x_ in d.detections)
        same += len(rs & got)
        tot += n
        got_n += len(got)
    r["dets"] = [same, tot, got_n]
    return r


def main():
    sd = seeded_sd(0)
    cases = []
    g = load_golden("detr_l_obj365_b2_640")
    cases.append(("golden_b2", synth_images(1, [(640, 640)] * 2), {k: g[k] for k in g.files}, 0.5))
    g = load_golden("detr_l_obj365_b3_ragged")
    cases.append(("golden_ragged", synth_images(2, [tuple(s) for s in g["image_sizes"].tolist()]), {k: g[k] for k in g.files}, float(g["threshold"])))
    # fresh inputs vs the CPU oracle
    imgs = synth_images(11, [(640, 640)] * 2)
    with torch.no_grad():
        ot = {}
        s, b = O.detr_forward(sd, O.detr_preprocess(imgs, (640, 640)), O.DetrOracleConfig(), ot)
        od = O.detr_postprocess(s, b, [(640, 640)] * 2, 0.5)
    od = [(list(d.boxes), list(d.labels)) for d in od]
    nmax = max(1, max(len(d[0]) for d in od))
    ref = {"scores": s.numpy(), "boxes": b.numpy(), "enc_topk_ind": ot["topk_ind"].numpy(), "det_count": np.array([len(d[0]) for d in od])}
    ref["det_labels"] = np.stack([np.pad(np.asarray(d[1], dtype=np.int64), (0, nmax - len(d[1]))) for d in od])
    ref["det_boxes"] = np.stack([np.pad(np.asarray(d[0], dtype=np.int64).reshape(-1, 4), ((0, nmax - len(d[0])), (0, 0))) for d in od])
    cases.append(("fresh_oracle", imgs, ref, 0.5))

    recipes = sys.argv[1:] or ["fp16", "fp32", "fp32_tc"]
    report = {}
    for rec in recipes:
        m = FAIDetr(DETRConfig(), precision=rec)
        m.load_state_dict(sd, strict=True)
        m.cuda()
        proc = DETRProcessor(m.config, image_size=640)
        report[rec] = {name: run_case(m, proc, imgs_, ref_, thr) for name, imgs_, ref_, thr in cases}
        for name in report[rec]:
            r = report[rec][name]
            print(f"{rec:8s} {name:14s} res3 {r.get('res3', float('nan')):.1e} res5 {r.get('res5', float('nan')):.1e} pan1 {r.get('pan1', float('nan')):.1e} "
                  f"overlap {r['overlap']} dscore {r['dscore']:.1e} dbox {r['dbox']:.1e} dets same/ref/got {r['dets']}", flush=True)
        del m
        torch.cuda.empty_cache()
    with open("error_budget.json", "w") as f:
        json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
