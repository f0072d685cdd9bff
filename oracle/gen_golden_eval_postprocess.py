"""Golden for DETRProcessor.eval_postprocess: the UNMODIFIED reference's `DETRProcessor.eval_postprocess` (models/fai_detr/processor.py) on the seeded
case of tests/test_eval_postprocess.py -> tests/golden/eval_postprocess.npz.  Needs the reference tree:  python -m oracle.gen_golden_eval_postprocess"""
import os

import numpy as np

from oracle import ref_import


def main():
    ref_import.install()
    from focoos.models.fai_detr.config import DETRConfig as RC
    from focoos.models.fai_detr.ports import DETRModelOutput as RO
    from focoos.models.fai_detr.processor import DETRProcessor as RP
    from focoos.nn.backbone.resnet import ResnetConfig as RB

    from tests.test_eval_postprocess import _case

    class Entry:  # DatasetEntry duck type
        def __init__(self, d):
            self.height, self.width = d["height"], d["width"]

    logits, boxes, entries = _case()
    ref = RP(RC(backbone_config=RB(), num_classes=20), image_size=640).eval_postprocess(RO(boxes=boxes.clone(), logits=logits.clone(), loss=None), [Entry(e) for e in entries], top_k=100)
    g = {}
    for i, r in enumerate(ref):
        inst = r["instances"]
        g[f"scores_{i}"] = inst.scores.numpy()
        g[f"classes_{i}"] = inst.classes.numpy()
        g[f"boxes_{i}"] = inst.boxes.tensor.numpy()
        g[f"image_size_{i}"] = np.array(tuple(inst.image_size), dtype=np.int64)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "eval_postprocess.npz")
    np.savez_compressed(path, n=np.array(len(ref)), **g)
    print("wrote", path)


if __name__ == "__main__":
    main()
