"""Goldens for the two comparisons with the UNMODIFIED reference that the tests used to make against a live import:
  * fai-detr-l-obj365 on one seeded 480x640 image: the reference's pre-processed input (SHA-256 and a seeded sample of 4096 values) and the per-image sorted
    max class logit of its 300 queries (tests/test_oracle.py::test_oracle_vs_live_reference);
  * `binary_mask_to_base64` (OpenCV PNG) on four seeded masks (tests/test_png_tail.py::test_against_the_live_reference_function).
-> tests/golden/live_reference.npz.  Needs the reference tree and OpenCV:  python -m oracle.gen_golden_live_reference"""
import hashlib
import os

import numpy as np
import torch

from oracle import ref_import
from oracle.gen_golden import synth_images
from tests.parity_utils import seeded_sd


def png_masks():
    rng = np.random.default_rng(11)
    return [rng.random(shape) > 0.6 for shape in ((1, 1), (5, 7), (120, 33), (64, 64))]


def x_sample_index(n):
    return np.sort(np.random.default_rng(5).choice(n, 4096, replace=False))


def main():
    ref_import.install()
    import cv2
    assert not type(cv2).__name__.startswith("_Dummy"), "OpenCV is needed to generate the goldens"
    from focoos.utils.vision import binary_mask_to_base64 as ref_fn

    fm = ref_import.get_reference_model("fai-detr-l-obj365")
    fm.model.load_state_dict(seeded_sd(0), strict=True)
    imgs = synth_images(7, [(480, 640)])
    with torch.no_grad():
        x, _ = fm.processor.preprocess(imgs, device=torch.device("cpu"), dtype=torch.float32)
        out = fm.model(x)
    xf = x.contiguous().numpy().ravel()
    g = {"x_sha256": np.array(hashlib.sha256(x.contiguous().numpy().tobytes()).hexdigest()), "x_shape": np.array(x.shape),
         "x_sample": xf[x_sample_index(xf.size)], "sorted_max_logit": np.sort(out.logits.numpy().max(-1), axis=1),
         "png_b64": np.array([ref_fn(m) for m in png_masks()])}
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "live_reference.npz")
    np.savez_compressed(path, **g)
    print("wrote", path)


if __name__ == "__main__":
    main()
