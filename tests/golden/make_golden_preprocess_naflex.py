"""Generate the SigLIP 2 NaFlex preprocessing fixture with transformers' `Siglip2ImageProcessorPil`.

    python tests/golden/make_golden_preprocess_naflex.py

Small seeded uint8 frames of several aspect ratios, patch 4, at two max_num_patches values: stores each frame and the
processor's pixel_values / pixel_attention_mask / spatial_shapes.  Needs transformers + Pillow (not needed where the tests run:
the .npz is committed).
"""
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import preprocess_oracle as P  # only for the seeded synthetic images

PATCH = 4
MAX_NUM_PATCHES = (16, 64)
SIZES = [(37, 53), (64, 64), (9, 70), (50, 11), (3, 5), (100, 75)]


def main():
    from transformers import Siglip2ImageProcessorPil

    data = {"patch": np.array(PATCH), "max_num_patches": np.array(MAX_NUM_PATCHES)}
    imgs = [P.synthetic_u8_images(1, h, w, seed=300 + i)[0] for i, (h, w) in enumerate(SIZES)]
    for i, img in enumerate(imgs):
        data[f"img{i}"] = img
    for n in MAX_NUM_PATCHES:
        proc = Siglip2ImageProcessorPil(patch_size=PATCH, max_num_patches=n)
        r = proc(images=[Image.fromarray(i) for i in imgs], return_tensors="np")
        data[f"pixel_values_{n}"] = np.asarray(r["pixel_values"], np.float32)
        data[f"pixel_attention_mask_{n}"] = np.asarray(r["pixel_attention_mask"], np.int32)
        data[f"spatial_shapes_{n}"] = np.asarray(r["spatial_shapes"], np.int64)
    path = os.path.join(HERE, "preprocess_siglip2_naflex.npz")
    np.savez_compressed(path, **data)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
