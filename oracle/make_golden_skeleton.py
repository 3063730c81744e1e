"""Generate tests/golden/skeleton_condition_{random,ref}.npz from the reference's OWN skeleton MDM._get_embeddings
(model/diffusion_skeleton.py:194-215, imported through oracle.ref_loader) -- run where the reference tree is installed:
python -m oracle.make_golden_skeleton
TEST INFRASTRUCTURE.  Weights: seeded random init of the conditioning path (portable: the tests regenerate it from the
seed) or the shipped checkpoint (tests using those need oracle/_ref/weights, else skip).  Inputs: make_skeleton_batch at
tests/skeleton_helpers.GOLDEN_CASES.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader as RL  # noqa: E402
from tests.skeleton_helpers import GOLDEN_CASES, skeleton_encoder_weights, skeleton_inputs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def reference_embeddings(sd, B, T, past_len):
    model, _, _ = RL.build_mdm_skeleton(state_dict=sd, diffusion_steps=1000, past_len=past_len, dropout=0)
    with torch.no_grad():
        return model._get_embeddings(*skeleton_inputs(B, T, past_len))


def main():
    os.makedirs(OUT, exist_ok=True)
    for source in ("random", "ref"):
        sd = skeleton_encoder_weights(source)
        out = {}
        for B, T, P in GOLDEN_CASES:
            emb, gt = reference_embeddings(sd, B, T, P)
            out["cond_%d_%d_%d" % (B, T, P)] = emb.numpy()
            out["gt_%d_%d_%d" % (B, T, P)] = gt.numpy()
        path = os.path.join(OUT, "skeleton_condition_%s.npz" % source)
        np.savez_compressed(path, **out)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
