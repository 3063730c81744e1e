"""CPU restatement of the skeleton model's conditioning encoder, MDM._get_embeddings of reference
model/diffusion_skeleton.py:194-215.  TEST INFRASTRUCTURE (see oracle/__init__.py); the encoder layers are
oracle.restate's.  Pinned against the reference class by tests/test_skeleton_condition.py (live where the reference tree
is installed, else through tests/golden/skeleton_condition_*.npz written by oracle/make_golden_skeleton.py)."""
import torch.nn.functional as F

from .restate import encoder


def mdm_skeleton_condition(sd, body, obj, zero_pose_obj, past_len, nhead=4, rotary=None, faithful=True):
    """body (T,B,J,3), obj (T,B,P,3) sequence-first, zero_pose_obj (B,P,3) -> cond (Tp,B,D), Tp = min(past_len, T):
    bodyEmbedding(body[:Tp]) + objEmbedding(obj[:Tp]) + shapeEmbedding(zero_pose_obj), positional encoding, encoder."""
    T, B = body.shape[:2]
    body, obj = body.reshape(T, B, -1)[:past_len], obj.reshape(T, B, -1)[:past_len]
    shp = F.linear(zero_pose_obj.reshape(1, B, -1), sd["shapeEmbedding.weight"], sd["shapeEmbedding.bias"])
    emb = F.linear(body, sd["bodyEmbedding.weight"], sd["bodyEmbedding.bias"]) \
        + F.linear(obj, sd["objEmbedding.weight"], sd["objEmbedding.bias"]) + shp
    emb = emb + sd["PositionalEmbedding.pe"][: emb.shape[0]]
    return encoder(sd, emb, nhead, rotary, faithful)
