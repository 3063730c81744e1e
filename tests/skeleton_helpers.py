"""Shared by the skeleton conditioning tests and oracle/make_golden_skeleton.py."""
from argparse import Namespace

import numpy as np
import torch

from interdiff_b200 import synthetic as S
from interdiff_b200 import weights as W
from tests.helpers import mdm_weights

# (B, T, past_len) of the golden cases: the shipped window (10 of 15 frames), a window past the 16-frame attention slab
# (17 of 30: two slabs), a clip shorter than past_len (Tp = T = 8)
GOLDEN_CASES = ((2, 15, 10), (3, 30, 17), (2, 8, 10))

SKELETON_ARGS = dict(embedding_dim=256, smpl_dim=63, num_joints=21, num_points=12, dropout=0.0, num_heads=4, ff_size=256,
                     activation="gelu", latent_usage="memory", past_len=10, future_len=25, cond_mask_prob=0, diffusion_steps=1000,
                     noise_schedule="cosine", sigma_small=True, weight_v=1)


def skeleton_encoder_weights(source="auto", seed=236):
    """mdm_weights('skeleton') + the conditioning path's tensors (encoder.layers.*, shapeEmbedding.*): exported checkpoint
    weights ('ref', skips if absent) or seeded init ('random'); 'auto' = ref if present."""
    sd = mdm_weights("skeleton", source)
    enc = None
    if source in ("ref", "auto"):
        enc = W.load_ref_weights("diffusion_skeleton_encoder")
        if enc is None and source == "ref":
            import pytest
            pytest.skip("exported encoder weights not present (oracle/export_skeleton_encoder.py)")
    if enc is None:
        enc = W.random_state_dict(W.skeleton_encoder_shapes(), seed)
    sd = dict(sd)
    sd.update({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in enc.items()})
    return sd


def skeleton_inputs(B, T, past_len=10):
    """eval_skeleton.py:114-118's tensors from make_skeleton_batch: body_gt (T,B,21,3), obj_gt (T,B,12,3), pose_gt (T,B,7),
    zero_pose_obj (B,12,3); the first three are transposed views of batch-first tensors, as the script passes them."""
    b = S.make_skeleton_batch(B=B, T=T, past_len=past_len)
    xs = torch.from_numpy(b["gt"]).squeeze(1).permute(2, 0, 1)            # (T,B,106)
    batch = [xs[..., :63].reshape(T, B, 21, 3).transpose(0, 1).contiguous(), xs[..., 63:99].reshape(T, B, 12, 3).transpose(0, 1).contiguous(),
             xs[..., 99:].transpose(0, 1).contiguous(), torch.from_numpy(b["zero_pose_obj"])]
    return batch[0].transpose(0, 1), batch[1].transpose(0, 1), batch[2].transpose(0, 1), batch[3]


def mirror_args(**over):
    return Namespace(**{**SKELETON_ARGS, **over})
