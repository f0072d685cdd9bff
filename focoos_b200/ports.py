"""Data classes mirrored from the reference's `focoos/ports.py` and `focoos/models/fai_detr/{ports,config}.py`
(only what the detection hot path exchanges with its callers)."""
from __future__ import annotations

from dataclasses import dataclass, field, fields
from typing import List, Optional, Union

import torch


@dataclass
class ModelOutput:
    """ports.py:875-920 (DictClass / ModelOutput): tuple view drops None fields, order = field order."""

    def to_tuple(self):
        return tuple(getattr(self, f.name) for f in fields(self) if getattr(self, f.name) is not None)


@dataclass
class DETRModelOutput(ModelOutput):
    """models/fai_detr/ports.py:9-13."""

    boxes: torch.Tensor  # [N, num_queries, 4] XYXY normalised to [0, 1]
    logits: torch.Tensor  # [N, num_queries, num_classes] sigmoid scores
    loss: Optional[dict] = None


@dataclass
class FocoosDet:
    """ports.py:303-356."""

    bbox: Optional[List[int]] = None
    conf: Optional[float] = None
    cls_id: Optional[int] = None
    label: Optional[str] = None
    mask: Optional[str] = None
    keypoints: Optional[list] = None


@dataclass
class FocoosDetections:
    """ports.py:373-420 (latency filled by the caller)."""

    detections: List[FocoosDet] = field(default_factory=list)
    latency: Optional[dict] = None

    def __len__(self):
        return len(self.detections)


class Boxes:
    """structures.py `Boxes`: an [N, 4] xyxy tensor (only what the evaluators read)."""

    def __init__(self, tensor: torch.Tensor):
        self.tensor = tensor

    def __len__(self):
        return int(self.tensor.shape[0])

    def to(self, *a, **k):
        return Boxes(self.tensor.to(*a, **k))


class Instances:
    """structures.py `Instances`: per-image prediction container with `image_size` = (height, width) and per-instance fields
    (`boxes: Boxes`, `scores`, `classes`), as consumed by the evaluators (trainer/evaluation/*)."""

    def __init__(self, image_size, **fields_):
        self.image_size = tuple(image_size)
        self._fields = dict(fields_)

    def __getattr__(self, name):
        f = self.__dict__.get("_fields", {})
        if name in f:
            return f[name]
        raise AttributeError(name)

    def has(self, name):
        return name in self._fields

    def get_fields(self):
        return self._fields

    def __len__(self):
        for v in self._fields.values():
            return len(v)
        return 0

    def to(self, *a, **k):
        return Instances(self.image_size, **{n: (v.to(*a, **k) if hasattr(v, "to") else v) for n, v in self._fields.items()})


@dataclass
class ResnetConfig:
    """nn/backbone/resnet.py:152-161."""

    in_chans: int = 3
    depth: int = 50
    variant: str = "d"
    freeze_at: int = -1
    num_stages: int = 4
    freeze_norm: bool = False
    model_type: str = "resnet"
    act: str = "relu"
    pretrained: bool = False
    use_pretrained: bool = False
    backbone_url: Optional[str] = None


@dataclass
class STDCConfig:
    """nn/backbone/stdc.py:175-186."""

    in_chans: int = 3
    base: int = 64
    layers: List[int] = field(default_factory=lambda: [4, 5, 3])
    out_features: List[str] = field(default_factory=lambda: ["res2", "res3", "res4", "res5"])
    model_type: str = "stdc"
    block_num: int = 4
    block_type: str = "cat"
    backbone_url: Optional[str] = None
    size: Optional[str] = None
    use_conv_last: bool = False
    use_pretrained: bool = False


_BACKBONE_CONFIGS = {"resnet": ResnetConfig, "stdc": STDCConfig}


def backbone_config_from_dict(bc, owner: str):
    """the trunk dataclass named by a registry `backbone_config` dict's model_type ("resnet" when absent); a dataclass passes through.
    `owner` names the model config in the error raised for an unknown model_type."""
    bc = bc or {}
    if not isinstance(bc, dict):
        return bc
    kind = bc.get("model_type", "resnet")
    if kind not in _BACKBONE_CONFIGS:
        raise ValueError(f"Invalid backbone model_type for {owner}: {kind!r} (expected one of {sorted(_BACKBONE_CONFIGS)})")
    bcls = _BACKBONE_CONFIGS[kind]
    return bcls(**{k: v for k, v in bc.items() if k in {f.name for f in fields(bcls)}})


@dataclass
class DETRConfig:
    """models/fai_detr/config.py:9-61 (same field names and defaults)."""

    backbone_config: Union[ResnetConfig, STDCConfig] = field(default_factory=ResnetConfig)
    num_classes: int = 365
    num_queries: int = 300
    resolution: Optional[int] = 640
    pixel_mean: List[float] = field(default_factory=lambda: [123.675, 116.28, 103.53])
    pixel_std: List[float] = field(default_factory=lambda: [58.395, 57.12, 57.375])
    size_divisibility: int = 0
    pixel_decoder_out_dim: int = 256
    pixel_decoder_feat_dim: int = 256
    pixel_decoder_num_encoder_layers: int = 1
    pixel_decoder_expansion: float = 1.0
    pixel_decoder_dim_feedforward: int = 1024
    transformer_predictor_out_dim: int = 256
    transformer_predictor_hidden_dim: int = 256
    transformer_predictor_dec_layers: int = 6
    transformer_predictor_dim_feedforward: int = 1024
    head_out_dim: int = 256
    pixel_decoder_dropout: float = 0.0
    pixel_decoder_nhead: int = 8
    transformer_predictor_nhead: int = 8
    threshold: float = 0.5
    top_k: int = 300
    # loss configuration (kept for config-file compatibility; training is a later round)
    criterion_deep_supervision: bool = True
    criterion_eos_coef: float = 0.1
    criterion_losses: List[str] = field(default_factory=lambda: ["vfl", "boxes"])
    criterion_num_points: int = 0
    criterion_focal_alpha: float = 0.75
    criterion_focal_gamma: float = 2.0
    weight_dict_loss_vfl: int = 1
    weight_dict_loss_bbox: int = 5
    weight_dict_loss_giou: int = 2
    matcher_cost_class: int = 2
    matcher_cost_bbox: int = 5
    matcher_cost_giou: int = 2
    matcher_use_focal_loss: bool = True
    matcher_alpha: float = 0.25
    matcher_gamma: float = 2.0

    def __post_init__(self):
        # the registry ships hybrid encoders with one AIFI layer (fai-detr-l-*) or none (fai-detr-m-coco); the engine runs exactly these two
        if self.pixel_decoder_num_encoder_layers not in (0, 1):
            raise ValueError(f"pixel_decoder_num_encoder_layers must be 0 or 1 (got {self.pixel_decoder_num_encoder_layers})")

    @classmethod
    def from_dict(cls, d: dict) -> "DETRConfig":
        d = dict(d)
        bc = backbone_config_from_dict(d.pop("backbone_config", {}), "DETRConfig")
        known = {f.name for f in fields(cls)}
        unknown = set(d) - known
        if unknown:
            raise ValueError(f"Invalid parameters for DETRConfig: {sorted(unknown)}")  # model_manager.py:376-381
        return cls(backbone_config=bc, **d)
