"""`model.export` of the CUDA path (SURVEY §8f.4) — mirror of `focoos/models/focoos_model.py:60-85,418-573` (ExportableModel, FocoosModel.export),
`focoos/infer/runtimes/torchscript.py:15-80` (TorchscriptRuntime) and the slice of `focoos/infer/infer_model.py` that serves an exported file.

The reference exports by `torch.jit.trace(ExportableModel(model), 128 * randn(1,3,H,W))`: a graph of ~1000 aten ops.  The CUDA engine is not a graph of
torch ops (its kernels are called through the C ABI), so the exported graph is ONE custom operator

    focoos_b200::model_forward(Tensor images, Tensor[] weights, str meta) -> Tensor[]

whose `weights` are the traced module's own parameters / buffers (so they are saved inside the `.pt`, follow `.to(device)`, and the file is
self-contained) and whose `meta` (JSON: family, config, precision, state_dict keys) lets the operator rebuild the engine on first use.  Loading the file
needs `import focoos_b200` first (it registers the operator - "the op library preloaded", torchscript.py:47-48 then works unchanged).  A fake
(meta-tensor) implementation is registered so that shape propagation / `torch.export` / FakeTensor tracing see correct output shapes.
"""
from __future__ import annotations

import json
import os
import time
from dataclasses import asdict, is_dataclass
from typing import List, Optional, Tuple, Union

import numpy as np
import torch
from torch import nn

from . import ops as _ops  # noqa: F401  (defines the focoos_b200:: operator namespace)

_LIB = torch.library.Library("focoos_b200", "FRAGMENT")  # the namespace is defined in ops.py
_LIB.define("model_forward(Tensor images, Tensor[] weights, str meta) -> Tensor[]")
_cache = {}


def _families():
    from .bisenetformer import BisenetFormer, BisenetFormerConfig
    from .fai_detr import FAIDetr
    from .fai_mf import FAIMaskFormer, MaskFormerConfig
    from .ports import DETRConfig
    return {"fai_detr": (DETRConfig, FAIDetr), "fai_mf": (MaskFormerConfig, FAIMaskFormer), "bisenetformer": (BisenetFormerConfig, BisenetFormer)}


def family_of(model) -> str:
    for name, (_, cls) in _families().items():
        if type(model) is cls:
            return name
    raise ValueError(f"{type(model).__name__} is not an exportable focoos_b200 model")


def make_meta(model) -> str:
    cfg = model.config
    return json.dumps({"family": family_of(model), "config": asdict(cfg) if is_dataclass(cfg) else dict(cfg), "precision": model.precision,
                       "keys": list(model.state_dict().keys())}, sort_keys=True)


def _rebuild(meta: str, weights: List[torch.Tensor]):
    info = json.loads(meta)
    cfg_cls, model_cls = _families()[info["family"]]
    m = model_cls(cfg_cls.from_dict(info["config"]), precision=info["precision"])
    res = m.load_state_dict(dict(zip(info["keys"], weights)))
    assert not res.missing_keys, res.missing_keys[:5]
    return m.to(weights[0].device).eval()


def _model_forward(images, weights, meta):
    key = (meta, str(images.device), tuple(int(w.data_ptr()) for w in weights[:4]), len(weights))
    m = _cache.get(key)
    if m is None:
        if len(_cache) >= 4:
            _cache.pop(next(iter(_cache)))
        m = _cache[key] = _rebuild(meta, list(weights))
    with torch.no_grad():
        out = m(images)
    return [t.contiguous() for t in out.to_tuple()]


_LIB.impl("model_forward", _model_forward, "CUDA")
_LIB.impl("model_forward", _model_forward, "CPU")  # reaches the models' own "CUDA only - no CPU fallback" error (or the tests' reference backend)


def output_shapes(meta: str, image_shape) -> List[Tuple[int, ...]]:
    """shapes of `model(images).to_tuple()` for an NCHW image batch: (boxes, logits) / (masks, logits)"""
    info = json.loads(meta)
    B, _, H, W = image_shape
    c = info["config"]
    if info["family"] == "fai_detr":
        return [(B, c["num_queries"], 4), (B, c["num_queries"], c["num_classes"])]
    return [(B, c["num_queries"], H, W), (B, c["num_queries"], c["num_classes"])]


@torch.library.register_fake("focoos_b200::model_forward")
def _model_forward_fake(images, weights, meta):
    return [images.new_empty(s, dtype=torch.float32) for s in output_shapes(meta, images.shape)]


class ExportableModel(nn.Module):
    """focoos_model.py:60-85: wraps the model for tracing, `forward(x) -> model(x).to_tuple()`."""

    def __init__(self, model, device="cuda", input_size=None):
        super().__init__()
        self.model = model.eval().to(device)
        self.meta = make_meta(self.model)

    def forward(self, x):
        weights = [t for _, t in self.model.state_dict(keep_vars=True).items()]
        out = torch.ops.focoos_b200.model_forward(x, weights, self.meta)
        return tuple(out[i] for i in range(len(output_shapes(self.meta, x.shape))))


class TorchscriptRuntime:
    """infer/runtimes/torchscript.py:15-80 for a file produced by `FocoosModel.export`: `__call__(im) -> tuple of tensors`, `benchmark`."""

    def __init__(self, model_path: str, model_info=None, device: str = "cuda", warmup_iter: int = 2):
        self.device = torch.device(device)
        self.model_info = model_info
        self.model = torch.jit.load(model_path, map_location=self.device)
        size = getattr(model_info, "im_size", None) or 640
        size = (size, size) if isinstance(size, int) else tuple(size)
        with torch.no_grad():
            for _ in range(warmup_iter):
                self.model(torch.rand(1, 3, *size, device=self.device))

    def __call__(self, im: torch.Tensor):
        with torch.no_grad():
            return self.model(im)

    def benchmark(self, iterations: int = 20, size: Union[int, Tuple[int, int]] = 640) -> dict:
        size = (size, size) if isinstance(size, int) else tuple(size)
        x = torch.rand(1, 3, *size, device=self.device)
        ts = []
        with torch.no_grad():
            for it in range(iterations + 5):
                t0 = time.perf_counter()
                self.model(x)
                torch.cuda.synchronize(self.device)
                if it >= 5:
                    ts.append((time.perf_counter() - t0) * 1e3)
        a = np.array(ts)
        return {"fps": int(1000 / a.mean()), "engine": "torchscript(focoos_b200)", "mean": round(float(a.mean()), 3), "min": round(float(a.min()), 3),
                "max": round(float(a.max()), 3), "std": round(float(a.std()), 3), "im_size": size[0], "device": str(self.device)}


class InferModel:
    """The part of infer/infer_model.py an exported detector needs: load the runtime + the processor, `infer(image) -> FocoosDetections`
    through `processor.export_postprocess` (infer_model.py:223-262)."""

    def __init__(self, model_path: str, model_info, processor, device: str = "cuda"):
        self.model_path, self.model_info, self.processor = model_path, model_info, processor
        self.runtime = TorchscriptRuntime(model_path, model_info, device)

    def infer(self, image, threshold: Optional[float] = None):
        im, _ = self.processor.preprocess(image, device=self.runtime.device, dtype=torch.float32)
        if im.dtype == torch.uint8:  # the exported graph takes the reference's float NCHW input
            im = im.permute(0, 3, 1, 2).float().contiguous()
        out = self.runtime(im)
        return self.processor.export_postprocess(out, image, class_names=getattr(self.model_info, "classes", ()) or (), threshold=threshold or 0.5)[0]

    __call__ = infer

    def benchmark(self, iterations: int = 20, size=None):
        return self.runtime.benchmark(iterations, size or getattr(self.model_info, "im_size", 640))


def export_model(focoos_model, runtime_type: str = "torchscript_32", out_dir: Optional[str] = None, device: str = "cuda", overwrite: bool = True,
                 image_size: Optional[Union[int, Tuple[int, int]]] = None) -> InferModel:
    """FocoosModel.export (focoos_model.py:418-573) for the TorchScript runtime types; ONNX / TensorRT are the reference's other backends and are not part
    of the CUDA path (ValueError, like the reference for unsupported formats)."""
    rt = str(getattr(runtime_type, "value", runtime_type)).lower()
    if "torchscript" not in rt:
        raise ValueError(f"focoos_b200 exports TorchScript only (got runtime_type={runtime_type!r}); ONNX/TensorRT belong to the reference's own runtimes")
    import copy
    info = focoos_model.model_info
    out_dir = out_dir or os.path.join(os.path.expanduser("~"), "FocoosAI", "models", info.name)
    os.makedirs(out_dir, exist_ok=True)
    size = image_size if image_size is not None else info.im_size
    h, w = (size, size) if isinstance(size, int) else tuple(size)
    out_file = os.path.join(out_dir, "model.pt")  # ArtifactName.PT
    info.im_size = size
    if overwrite or not os.path.exists(out_file):
        exportable = ExportableModel(copy.deepcopy(focoos_model.model), device=device, input_size=size)
        data = 128 * torch.randn(1, 3, h, w, device=device)
        with torch.no_grad():
            exportable(data)  # warm-up, as the reference ("record the spatial shapes")
            traced = torch.jit.trace(exportable, data, check_trace=False)
        torch.jit.save(traced, out_file)
    with open(os.path.join(out_dir, "model_info.json"), "w") as f:  # ArtifactName.INFO
        json.dump({k: v for k, v in asdict(info).items()}, f, indent=1, default=str)
    return InferModel(out_file, info, focoos_model.processor, device)
