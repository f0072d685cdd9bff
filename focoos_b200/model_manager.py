"""ModelManager / FocoosModel — the reference's L5 facade for the detection hot path
(`focoos/model_manager.py:43-91`, `focoos/models/focoos_model.py:100,370,575`).

`ModelManager.get(name)` builds the H100-native model from the same registry JSON the reference ships
(`focoos/model_registry/<name>.json`, `config` section; a copy of the architecture section for the fai-detr
family is embedded below since the reference tree is not present on the GPU box).  No network: weights come from
`model_info["weights_path"]`, an explicit `state_dict=` argument, or stay at their initial values.
"""
from __future__ import annotations

import os
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import ops
from .bisenetformer import BisenetFormer, BisenetFormerConfig
from .fai_detr import FAIDetr
from .fai_mf import FAIMaskFormer, MaskFormerConfig
from .ports import DETRConfig, FocoosDetections
from .processor import DETRProcessor, MaskFormerProcessor

# architecture sections of focoos/model_registry/fai-detr-*.json (config.*; class lists omitted)
_REGISTRY: Dict[str, dict] = {
    "fai-detr-l-obj365": {"im_size": 640, "config": {"num_classes": 365, "backbone_config": {"model_type": "resnet", "depth": 50, "variant": "d"}, "num_queries": 300,
                                                     "resolution": 640, "threshold": 0.5}},
    "fai-detr-l-coco": {"im_size": 640, "config": {"num_classes": 80, "backbone_config": {"model_type": "resnet", "depth": 50, "variant": "d"}, "num_queries": 300,
                                                   "resolution": 640, "threshold": 0.5}},
    "fai-detr-m-coco": {"im_size": 640, "config": {"num_classes": 80, "backbone_config": {"model_type": "stdc", "in_chans": 3, "base": 64, "layers": [4, 5, 3],
                                                                            "out_features": ["res2", "res3", "res4", "res5"], "block_num": 4,
                                                                            "block_type": "cat", "use_conv_last": False},
                                                   "num_queries": 300, "resolution": 640, "pixel_decoder_out_dim": 128, "pixel_decoder_feat_dim": 128,
                                                   "pixel_decoder_num_encoder_layers": 0, "pixel_decoder_expansion": 1.0, "pixel_decoder_dim_feedforward": 1024,
                                                   "transformer_predictor_out_dim": 128, "transformer_predictor_hidden_dim": 256,
                                                   "transformer_predictor_dec_layers": 3, "transformer_predictor_dim_feedforward": 1024, "head_out_dim": 128,
                                                   "pixel_decoder_nhead": 8, "transformer_predictor_nhead": 8, "threshold": 0.5}},
    "fai-mf-l-coco-ins": {"family": "fai_mf", "im_size": 1024, "config": {"num_classes": 80, "backbone_config": {"model_type": "resnet", "depth": 101, "variant": "d"},
                                                                           "num_queries": 100, "postprocessing_type": "instance", "predict_all_pixels": False,
                                                                           "use_mask_score": True, "threshold": 0.5}},
    **{name: {"family": "fai_mf", "im_size": 1024, "config": {"num_classes": 80, "backbone_config": {"model_type": "resnet", "depth": depth, "variant": "d"},
                                                             "num_queries": 100, "resolution": 1024, "pixel_decoder_out_dim": 128, "pixel_decoder_feat_dim": 128,
                                                             "pixel_decoder_transformer_layers": 3, "pixel_decoder_transformer_nheads": 8,
                                                             "pixel_decoder_transformer_dim_feedforward": 1024, "transformer_predictor_out_dim": 128,
                                                             "transformer_predictor_hidden_dim": 256, "transformer_predictor_dec_layers": 6,
                                                             "transformer_predictor_dim_feedforward": 1024, "head_out_dim": 128, "postprocessing_type": "instance",
                                                             "predict_all_pixels": False, "use_mask_score": True, "threshold": 0.5}}
       for name, depth in (("fai-mf-m-coco-ins", 101), ("fai-mf-s-coco-ins", 50))},
    "bisenetformer-l-ade": {"family": "bisenetformer", "im_size": 640, "config": {"num_classes": 150, "backbone_config": {"model_type": "stdc", "base": 64, "layers": [4, 5, 3]},
                                                                                   "num_queries": 100, "postprocessing_type": "semantic", "predict_all_pixels": True,
                                                                                   "use_mask_score": False, "threshold": 0.5}},
    # ADE20K semantic MaskFormers: no pixel-decoder encoder (layer_4 reads res5), ResNet-101-vd (-l) or STDC-2 (-m) trunk
    **{name: {"family": "fai_mf", "im_size": 640, "config": {"num_classes": 150, "backbone_config": bc, "num_queries": 100, "resolution": 640,
                                                            "pixel_decoder_out_dim": 128, "pixel_decoder_feat_dim": 128, "pixel_decoder_transformer_layers": 0,
                                                            "pixel_decoder_transformer_nheads": 8, "pixel_decoder_transformer_dim_feedforward": 1024,
                                                            "transformer_predictor_out_dim": 128, "transformer_predictor_hidden_dim": 256,
                                                            "transformer_predictor_dec_layers": dec_layers, "transformer_predictor_dim_feedforward": dff,
                                                            "head_out_dim": 128, "postprocessing_type": "semantic", "mask_threshold": 0.5, "predict_all_pixels": True,
                                                            "use_mask_score": False, "threshold": 0.5, "top_k": 100}}
       for name, bc, dec_layers, dff in (
           ("fai-mf-l-ade", {"model_type": "resnet", "depth": 101, "variant": "d"}, 6, 1024),
           ("fai-mf-m-ade", {"model_type": "stdc", "in_chans": 3, "base": 64, "layers": [4, 5, 3], "out_features": ["res2", "res3", "res4", "res5"],
                             "block_num": 4, "block_type": "cat", "use_conv_last": False}, 3, 512))},
    # ADE20K BisenetFormers: -m has a 96-wide pixel decoder and 4 decoder layers, -s the STDC-1 trunk (layers [2, 2, 2])
    **{name: {"family": "bisenetformer", "im_size": 640, "config": {"num_classes": 150, "backbone_config": {"model_type": "stdc", "in_chans": 3, "base": 64, "layers": layers,
                                                                                                           "out_features": ["res2", "res3", "res4", "res5"], "block_num": 4,
                                                                                                           "block_type": "cat", "use_conv_last": False},
                                                                   "num_queries": 100, "pixel_decoder_out_dim": width, "pixel_decoder_feat_dim": width,
                                                                   "transformer_predictor_out_dim": width, "transformer_predictor_hidden_dim": 256,
                                                                   "transformer_predictor_dec_layers": dec_layers, "transformer_predictor_dim_feedforward": dff,
                                                                   "head_out_dim": width, "postprocessing_type": "semantic", "top_k": 100, "mask_threshold": 0.5,
                                                                   "predict_all_pixels": True, "use_mask_score": False, "threshold": 0.5}}
       for name, layers, width, dec_layers, dff in (("bisenetformer-m-ade", [4, 5, 3], 96, 4, 512), ("bisenetformer-s-ade", [2, 2, 2], 128, 6, 1024))},
}

# model family -> (config class, nn.Module class, processor class, resize inputs to im_size?) — ModelManager.register_model / ProcessorManager
# (focoos/model_manager.py:94-105, focoos/processor/processor_manager.py:14-18)
_FAMILIES = {
    "fai_detr": (DETRConfig, FAIDetr, DETRProcessor, True),
    "fai_mf": (MaskFormerConfig, FAIMaskFormer, MaskFormerProcessor, False),
    "bisenetformer": (BisenetFormerConfig, BisenetFormer, MaskFormerProcessor, False),
}


@dataclass
class ModelInfo:
    name: str
    model_family: str = "fai_detr"
    classes: List[str] = field(default_factory=list)
    im_size: int = 640
    config: dict = field(default_factory=dict)
    weights_uri: Optional[str] = None


class FocoosModel:
    """focoos_model.py:100: owns the nn.Module + processor; `infer` / `__call__` / `benchmark`."""

    def __init__(self, model, model_info: ModelInfo):
        self.model, self.model_info = model, model_info
        _, _, proc_cls, resize = _FAMILIES[model_info.model_family]
        self.processor = proc_cls(model.config, image_size=model_info.im_size if resize else None).eval()
        self.model.eval()
        if torch.cuda.is_available() and ops._backend is None:  # the tests' CPU reference operators take host tensors only
            self.model.cuda()
        # CUDA-graph cache of model.forward per (input shape, dtype): the eager forward is ~240 launches of partly very short kernels (the
        # decoder runs ahead of a Python host), so replaying a captured graph removes the host from the critical path of `infer` / `__call__`
        self.cuda_graphs = os.environ.get("FB200_NO_GRAPH", "0") != "1"
        self._graphs = {}  # key -> (graph, static_input, static_output, the engine whose packed weights the graph reads)
        self._graph_seen = {}
        self._pipe = None  # infer_async state: copy stream, two staging / pinned result buffers

    def _forward(self, images):
        """model.forward, through a cached CUDA graph when the same input shape has been seen before (first sighting runs eagerly)."""
        if not (self.cuda_graphs and images.is_cuda and ops._backend is None):
            return self.model(images)
        key = (tuple(images.shape), images.dtype, getattr(self.model, "precision", None), bool(getattr(self.model, "lazy_masks", False)))
        ent = self._graphs.get(key)
        if ent is not None and ent[3] is not getattr(self.model, "_engine", None):
            # the model re-packed its weights (load_state_dict / train() -> eval() / .to()): the captured graph points at the OLD packed tensors
            # (kept alive by the entry, so the replay would be valid but stale) - drop it and capture again
            del self._graphs[key]
            ent = None
            self._graph_seen[key] = 1
        if ent is None:
            self._graph_seen[key] = self._graph_seen.get(key, 0) + 1
            if self._graph_seen[key] < 2:  # capture only shapes that come back (a one-off image size is not worth 2+ GB of pooled activations)
                return self.model(images)
            if len(self._graphs) >= 2:  # bounded: each entry owns a private activation pool
                self._graphs.pop(next(iter(self._graphs)))
            static_in = images.clone()
            self.model(static_in)  # make sure every lazily-initialised piece (engine, constants) exists before capture
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self.model(static_in)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            with torch.cuda.graph(g):
                static_out = self.model(static_in)
            ent = self._graphs[key] = (g, static_in, static_out, getattr(self.model, "_engine", None))
        g, static_in, static_out, _ = ent
        static_in.copy_(images, non_blocking=True)
        g.replay()
        return static_out

    @property
    def device(self):
        return self.model.device

    def __call__(self, inputs, threshold: Optional[float] = None, batched: bool = False):
        """focoos_model.py:575-621.  The reference returns only the first image's detections ("we don't support
        batching yet", :615-621); `batched=True` returns all of them (SURVEY §8f.1)."""
        t0 = time.perf_counter()
        images, _ = self.processor.preprocess(inputs, device=self.device, dtype=torch.float32)
        t1 = time.perf_counter()
        with torch.no_grad():
            # segmentation families: let the processor fuse the final mask upsampling into its own reduction (fai_mf.LazyMasks)
            fused = hasattr(self.model, "lazy_masks")
            if fused:
                self.model.lazy_masks = True
            try:
                out = self._forward(images)
            finally:
                if fused:
                    self.model.lazy_masks = False
        t2 = time.perf_counter()
        dets = self.processor.postprocess(out, inputs, class_names=self.model_info.classes, threshold=threshold)
        t3 = time.perf_counter()
        lat = {"preprocess": round(t1 - t0, 3), "inference": round(t2 - t1, 3), "postprocess": round(t3 - t2, 3)}
        for d in dets:
            d.latency = lat
        return dets if batched else dets[0]

    # ---- pipelined inference (SURVEY §8f.1): the host edge overlapped with the device ------------------------------------------------
    def infer_async(self, inputs, threshold: Optional[float] = None) -> "PendingDetections":
        """Enqueue one batch and return at once; `.result()` yields what `self(inputs, batched=True)` would.

        fai-detr family with a pinned uint8 [B,H,W,3] batch at the model resolution: the H2D copy runs on a COPY stream into one of two staging
        buffers, the compute stream then (a) copies staging -> the CUDA graph's static input (device to device), (b) replays the graph, (c) runs the
        fused post-process, (d) sends the packed detections to one of two pinned host buffers.  Nothing blocks the host, so the copy of batch k+1
        and the Python-side object building of batch k-1 overlap with the device work of batch k.  Any other input takes the synchronous path."""
        from .processor import _is_u8_nhwc_batch
        fast = (isinstance(self.processor, DETRProcessor) and type(self.processor) is DETRProcessor and _is_u8_nhwc_batch(inputs) and not inputs.is_cuda
                and self.cuda_graphs and ops._backend is None and self.model.device.type == "cuda")
        if fast:
            tgt = self.processor.image_size
            tgt = (tgt, tgt) if isinstance(tgt, int) else tgt
            fast = tgt is None or tuple(inputs.shape[1:3]) == tuple(tgt)
        if not fast:
            return PendingDetections(ready=self(inputs, threshold=threshold, batched=True))
        dev = self.model.device
        st = self._pipe
        key = (tuple(inputs.shape), getattr(self.model, "precision", None))
        if st is None or st["key"] != key:
            B = inputs.shape[0]
            K = self.processor.top_k
            st = self._pipe = {"key": key, "copy": torch.cuda.Stream(device=dev), "k": 0,
                               "staging": [torch.empty(inputs.shape, dtype=torch.uint8, device=dev) for _ in range(2)],
                               "host": [torch.empty((B, K * 7 + 1), dtype=torch.int32).pin_memory() for _ in range(2)],
                               "h2d_done": [torch.cuda.Event() for _ in range(2)], "free": [torch.cuda.Event() for _ in range(2)],
                               "sizes": torch.tensor([(int(inputs.shape[1]), int(inputs.shape[2]))] * B, dtype=torch.int32, device=dev)}
            for _ in range(2):  # first sighting runs eagerly, the second captures the graph (see _forward)
                self._forward(st["staging"][0])
            torch.cuda.synchronize(dev)
        k = st["k"] & 1
        st["k"] += 1
        cur = torch.cuda.current_stream(dev)
        with torch.cuda.stream(st["copy"]):
            st["copy"].wait_event(st["free"][k])       # the compute stream has finished reading this staging buffer (two batches ago)
            st["staging"][k].copy_(inputs, non_blocking=True)
            st["h2d_done"][k].record(st["copy"])
        cur.wait_event(st["h2d_done"][k])
        with torch.no_grad():
            out = self._forward(st["staging"][k])      # static_in.copy_(staging) + graph replay, all on the compute stream
            st["free"][k].record(cur)
            packed = self.processor.postprocess_packed(out, None, None, threshold, sizes_dev=st["sizes"])
            st["host"][k].copy_(packed, non_blocking=True)
        done = torch.cuda.Event()
        done.record(cur)
        return PendingDetections(event=done, host=st["host"][k], class_names=self.model_info.classes)

    def stream(self, batches, threshold: Optional[float] = None, depth: int = 2):
        """generator over an iterable of batches: yields each batch's detections, keeping `depth` batches in flight (see infer_async)"""
        from collections import deque
        q = deque()
        for b in batches:
            q.append(self.infer_async(b, threshold))
            if len(q) >= depth:
                yield q.popleft().result()
        while q:
            yield q.popleft().result()

    # ---- export / train / eval (focoos_model.py:418-573, 221-275, 276-310) ------------------------------------------------------------
    def export(self, runtime_type="torchscript_32", onnx_opset: int = 18, out_dir: Optional[str] = None, device: str = "auto", simplify_onnx: bool = True,
               overwrite: bool = True, image_size=None, dynamic_axes: bool = True):
        """focoos_model.py:418-573 for the TorchScript runtimes: `torch.jit.trace(ExportableModel)` -> `<out_dir>/model.pt` + `model_info.json`, returns an
        InferModel serving the file.  The traced graph is one `focoos_b200::model_forward` operator over the module's own weights (focoos_b200/export.py);
        reloading it reproduces the eager outputs bit for bit.  ONNX / TensorRT runtime types raise ValueError (the reference's other backends)."""
        from .export import export_model
        dev = ("cuda" if torch.cuda.is_available() else "cpu") if device == "auto" else device
        return export_model(self, runtime_type, out_dir, dev, overwrite, image_size)

    def train(self, args, data_train, data_val=None, hub=None):
        """focoos_model.py:221-275: fine-tune on `data_train` (single process, or `args.num_gpus` processes with the NCCL gradient exchange), write
        `<output_dir>/<run_name>/model_final.pth` + `model_info.json`, reload the trained weights and return to eval mode."""
        from .trainer import run_train_entry
        assert hub is None, "Focoos Hub sync is outside the CUDA hot path"
        return run_train_entry(self, args, data_train, data_val)

    def eval(self, args, data_test, save_json: bool = True):
        """focoos_model.py:276-310: `inference_on_dataset` with `processor.eval_postprocess` and the processor's evaluator (box AP for fai-detr, mIoU for semantic
        segmenters); returns the metrics dict."""
        from .trainer import run_eval_entry
        return run_eval_entry(self, args, data_test, save_json)

    def infer(self, image, threshold: Optional[float] = None) -> FocoosDetections:
        """focoos_model.py:370: single image (ndarray HWC uint8 / PIL / tensor) -> FocoosDetections."""
        return self(image, threshold=threshold)

    def benchmark(self, iterations: int = 50, size=(640, 640), batch: int = 1) -> dict:
        """BaseModelNN.benchmark (models/base_model.py:160-216): CUDA-event latency of model.forward on 128*randn input."""
        x = 128 * torch.randn(batch, 3, size[0], size[1], device=self.device)
        for _ in range(5):
            self.model(x)
        torch.cuda.synchronize()
        ts = []
        for _ in range(iterations):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            self.model(x)
            e.record()
            e.synchronize()
            ts.append(s.elapsed_time(e))
        a = np.array(ts)
        return {"fps": int(1000 * batch / a.mean()), "mean": round(float(a.mean()), 3), "min": round(float(a.min()), 3), "max": round(float(a.max()), 3),
                "std": round(float(a.std()), 3), "im_size": size[0], "device": str(self.device), "engine": "focoos_b200"}


class PendingDetections:
    """handle returned by FocoosModel.infer_async: `.result()` waits for the device (one event) and builds the FocoosDetections"""

    def __init__(self, ready=None, event=None, host=None, class_names=()):
        self._ready, self._event, self._host, self._names = ready, event, host, class_names

    def result(self) -> List[FocoosDetections]:
        if self._ready is None:
            self._event.synchronize()
            # the pinned buffer is reused two batches later: parse it now
            self._ready = DETRProcessor.detections_from_packed(self._host.numpy().copy(), self._names)
        return self._ready


class ModelManager:
    @classmethod
    def get(cls, name: str, model_info: Optional[ModelInfo] = None, config: Optional[DETRConfig] = None, state_dict=None,
            precision: str = "fp16", **kwargs) -> FocoosModel:
        """model_manager.py:43-91.  `kwargs` override config fields (validated like ConfigManager.from_dict, :336-389)."""
        if model_info is None:
            if name not in _REGISTRY:
                raise ValueError(f"Model {name} not found in the focoos_b200 registry ({sorted(_REGISTRY)})")
            r = _REGISTRY[name]
            model_info = ModelInfo(name=name, model_family=r.get("family", "fai_detr"), im_size=r["im_size"], config=dict(r["config"]))
        if model_info.model_family not in _FAMILIES:
            raise ValueError(f"Model family {model_info.model_family} is not on the CUDA hot path ({sorted(_FAMILIES)})")
        cfg_cls, model_cls, _, _ = _FAMILIES[model_info.model_family]
        if config is None:
            cd = dict(model_info.config)
            cd.update(kwargs)
            config = cfg_cls.from_dict(cd)
        model = model_cls(config, precision=precision)
        if state_dict is not None:
            model.load_state_dict(state_dict)
        elif model_info.weights_uri:
            model.load_state_dict(torch.load(model_info.weights_uri, map_location="cpu", weights_only=True))
        return FocoosModel(model, model_info)
