"""Deterministic, non-degenerate random weights for parity tests and benchmarks.

No pretrained checkpoint is reachable offline and the reference's default init is degenerate
(zero sampling-offset / attention-weight / bbox-head weights, identity BN statistics: every score
< 0.03, see SURVEY.md §8c).  `seeded_state_dict` re-randomises *every* tensor of a `state_dict`
from its NAME and SHAPE only (one CPU generator per key, seeded by crc32(name) ^ seed), so the
reference model (in the oracle container) and this project's model (on the GPU) get bit-identical
weights without shipping a 176 MB file.  CPU `torch.randn`/`rand` with a fixed generator seed is
reproducible for a fixed torch build (same image on both sides).
"""
from __future__ import annotations

import math
import zlib
from typing import Dict, Mapping, Sequence

import torch


def _gen(name: str, seed: int) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    return g


def _uniform(shape, lo, hi, g):
    return torch.rand(shape, generator=g, dtype=torch.float32) * (hi - lo) + lo


def _normal(shape, std, g, mean=0.0):
    return torch.randn(shape, generator=g, dtype=torch.float32) * std + mean


def seeded_tensor(name: str, shape: Sequence[int], dtype: torch.dtype, keys: Mapping[str, object], seed: int) -> torch.Tensor:
    g = _gen(name, seed)
    shape = tuple(shape)
    leaf = name.rsplit(".", 1)[-1]
    parent = name.rsplit(".", 1)[0] if "." in name else ""
    if not dtype.is_floating_point:  # num_batches_tracked
        return torch.zeros(shape, dtype=dtype)
    is_bn = (parent + ".running_mean") in keys
    if leaf == "running_mean":
        return _uniform(shape, -0.2, 0.2, g)
    if leaf == "running_var":
        return _uniform(shape, 0.5, 1.5, g)
    if leaf == "empty_weight":
        w = torch.ones(shape)
        w[-1] = 0.1
        return w
    if leaf == "weight" and len(shape) == 1:  # BN gamma / LN gamma
        if is_bn and (".branch2c." in name or name.endswith("bottlenecks.2.conv1.norm.weight") or name.endswith("bottlenecks.2.conv2.norm.weight")):
            return _uniform(shape, 0.25, 0.45, g)  # damp residual-branch growth
        return _uniform(shape, 0.8, 1.2, g)
    if leaf == "bias" and len(shape) == 1:
        if "score_classifier" in name or name.endswith("classifier.bias"):
            return _normal(shape, 1.0, g, mean=-8.0)  # spread of class priors -> scores straddle the 0.5 threshold
        if "sampling_offsets" in name:
            return _uniform(shape, -2.0, 2.0, g)
        if is_bn or (parent + ".weight") in keys and len(tuple(getattr(keys[parent + ".weight"], "shape", ()))) == 1:
            return _uniform(shape, -0.1, 0.1, g)  # norm beta
        return _uniform(shape, -0.1, 0.1, g)
    if leaf in ("weight", "in_proj_weight") and len(shape) == 4:  # conv [Co,Ci,kh,kw]
        fan_in = shape[1] * shape[2] * shape[3]
        return _normal(shape, math.sqrt(2.0 / fan_in), g)
    if leaf in ("weight", "in_proj_weight") and len(shape) == 2:  # linear / embedding
        fan_in = shape[1]
        std = math.sqrt(1.0 / fan_in)
        if "sampling_offsets" in name:
            std *= 0.5
        if "score_classifier" in name:
            std *= 2.5  # wide logit spread: the top-300 scores straddle the 0.5 threshold
        if name.endswith("forward_prediction_heads.classifier.weight"):
            std *= 3.0  # peaky class softmax so that some queries clear the 0.5 score threshold (MaskFormer family)
        if name.endswith("mask_classifier.layers.2.weight"):
            std *= 0.03  # keep mask logits O(10): mask_embed . mask_features sums 256 products of O(1..30) features
        if "bbox_classifier" in name and name.endswith("layers.2.weight"):
            std *= 0.5
        if name.endswith("query_feat.weight") or name.endswith("query_embed.weight"):
            std = 1.0
        return _normal(shape, std, g)
    if leaf == "in_proj_bias":
        return _uniform(shape, -0.1, 0.1, g)
    return _normal(shape, 0.02, g)


def seeded_state_dict(template: Mapping[str, torch.Tensor], seed: int = 0) -> Dict[str, torch.Tensor]:
    """Return a new state_dict with the same keys/shapes/dtypes as `template`, fully re-randomised."""
    out = {}
    for k, v in template.items():
        out[k] = seeded_tensor(k, v.shape, v.dtype, template, seed)
    return out


def desaturate_classifiers(sd, factor: float = 0.25):
    """Training-parity fixtures only: scale every score classifier (weights and biases) so that logits stay within a few units.
    The reference's matching cost contains -log(1 - sigmoid(x) + 1e-8) (fai_detr/modelling.py:733-735); for x in ~[15, 17] the fp32
    value of sigmoid(x) is either 1 or 1 - 2^-24 depending on the last ulp of exp(-x), which moves that term by ~2.5 - so with the
    saturated logits of the inference fixtures (up to 18) the Hungarian assignment is not reproducible between ANY two fp32
    implementations (torch CPU vs torch CUDA included).  Trained checkpoints do not reach that range."""
    out = dict(sd)
    for k, v in sd.items():
        if "score_classifier" in k:
            out[k] = v * factor
    return out
