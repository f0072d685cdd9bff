"""focoos_b200 — H100-native (sm_90a) implementation of the FocoosAI/focoos detection hot path."""
from .bisenetformer import BisenetFormer, BisenetFormerConfig  # noqa: F401
from .fai_detr import FAIDetr  # noqa: F401
from .fai_mf import FAIMaskFormer, MaskFormerConfig  # noqa: F401
from .model_manager import FocoosModel, ModelInfo, ModelManager  # noqa: F401
from .ports import DETRConfig, DETRModelOutput, FocoosDet, FocoosDetections, ResnetConfig  # noqa: F401
from .processor import DETRProcessor, MaskFormerProcessor  # noqa: F401

__version__ = "0.1.0"
