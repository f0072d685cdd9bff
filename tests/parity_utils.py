"""Helpers shared by the parity tests (test infrastructure)."""
from __future__ import annotations

import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def update_report(name: str, entries: dict):
    """merge `entries` into the JSON parity report `name` under $FB200_REPORT_DIR (default: a directory in the system temp dir), outside the source tree"""
    import tempfile
    d = os.environ.get("FB200_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "focoos_b200_reports")
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, name)
    rep = json.load(open(path)) if os.path.exists(path) else {}
    rep.update(entries)
    with open(path, "w") as f:
        json.dump(rep, f, indent=1)


def load_golden(tag: str):
    return np.load(os.path.join(GOLDEN, tag + ".npz"))


def golden_meta():
    with open(os.path.join(GOLDEN, "golden_meta.json")) as f:
        return json.load(f)


def manifest_template(name="fai_detr_l_obj365"):
    with open(os.path.join(GOLDEN, f"{name}_state_dict_manifest.json")) as f:
        man = json.load(f)
    return {k: torch.empty(v[0], dtype=getattr(torch, v[1])) for k, v in man.items()}


def seeded_sd(seed=0, name="fai_detr_l_obj365"):
    from focoos_b200.utils.seeded_weights import seeded_state_dict

    return seeded_state_dict(manifest_template(name), seed)


class ConvCalls:
    """ops backend wrapper that records the weight operand of every conv2d / conv2d_pair call (which flow a layer took)"""

    def __init__(self, be):
        self.be, self.w = be, {"conv2d": [], "conv2d_pair": []}

    def __getattr__(self, name):
        fn = getattr(self.be, name)
        if name not in self.w:
            return fn

        def call(*a):
            self.w[name].append(a[1])
            return fn(*a)
        return call


def align_by_key(key_a: np.ndarray, key_b: np.ndarray) -> np.ndarray:
    """perm such that key_b[perm] == key_a (both are permutations of the same unique set)."""
    assert sorted(key_a.tolist()) == sorted(key_b.tolist()), "query SETS differ"
    assert len(set(key_a.tolist())) == len(key_a)
    pos = {int(k): i for i, k in enumerate(key_b.tolist())}
    return np.array([pos[int(k)] for k in key_a.tolist()], dtype=np.int64)


def compare_queries(scores_a, boxes_a, key_a, scores_b, boxes_b, key_b):
    """Max abs diff of per-query scores / boxes after aligning rows by encoder anchor index.
    The encoder top-k ORDER is not comparable between two fp32 implementations (gaps between adjacent kept
    scores go down to 0, see golden 'enc_topk_val'); the selected SET and every per-anchor output are."""
    ds, db = 0.0, 0.0
    for i in range(scores_a.shape[0]):
        perm = align_by_key(np.asarray(key_a[i]), np.asarray(key_b[i]))
        ds = max(ds, float(np.abs(np.asarray(scores_a[i]) - np.asarray(scores_b[i])[perm]).max()))
        db = max(db, float(np.abs(np.asarray(boxes_a[i]) - np.asarray(boxes_b[i])[perm]).max()))
    return ds, db


def detections_match(det_a, det_b, score_tol=1e-4, box_tol=1):
    """det_* = (boxes int [n,4], scores [n], labels [n]) sorted by descending score.
    Class indices and keep-set must be identical; order may differ only inside score ties (< score_tol)."""
    ba, sa, la = det_a
    bb, sb, lb = det_b
    assert len(sa) == len(sb), f"keep-set size differs: {len(sa)} vs {len(sb)}"
    ka = sorted(zip(la.tolist(), map(tuple, ba.tolist())))
    kb = sorted(zip(lb.tolist(), map(tuple, bb.tolist())))
    if box_tol == 0:
        assert ka == kb, "keep-sets differ"
    else:
        assert [k[0] for k in ka] == [k[0] for k in kb], "class indices differ"
    assert np.abs(np.sort(sa) - np.sort(sb)).max() <= score_tol if len(sa) else True
    # order: a position may only be swapped with a neighbour whose score is within tol
    for i in range(len(sa)):
        if la[i] != lb[i] or tuple(ba[i]) != tuple(bb[i]):
            j = [j for j in range(len(sb)) if lb[j] == la[i] and np.abs(np.array(bb[j]) - np.array(ba[i])).max() <= box_tol and abs(sb[j] - sa[i]) <= score_tol]
            assert j, f"detection {i} of A has no counterpart in B"
    return True
