"""Export the skeleton model's conditioning tensors (encoder.layers.*, shapeEmbedding.*) of the reference's
checkpoints/diffusion_skeleton.ckpt to oracle/_ref/weights/diffusion_skeleton_encoder.npz (a build product, not in git),
next to the files of oracle/export_ref_weights.py.  TEST INFRASTRUCTURE.
Run where the reference tree is installed:  python -m oracle.export_skeleton_encoder
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200 import weights as W  # noqa: E402
from oracle import ref_loader as RL  # noqa: E402

NAME = "diffusion_skeleton_encoder"


def main():
    os.makedirs(W.REF_WEIGHT_DIR, exist_ok=True)
    _, sd = RL.load_ckpt("diffusion_skeleton")
    sel = {}
    for k, shp in W.skeleton_encoder_shapes().items():
        v = sd[k].numpy()
        assert tuple(v.shape) == tuple(shp), (k, v.shape, shp)
        sel[k] = v
    np.savez(W.ref_weights_path(NAME), **sel)
    print(NAME, len(sel), "tensors", sum(v.size for v in sel.values()) * 4 / 1e6, "MB")


if __name__ == "__main__":
    main()
