"""The skeleton model's conditioning encoder, MDM._get_embeddings (reference model/diffusion_skeleton.py:194-215), on the
CPU: the restatement oracle.skeleton_condition.mdm_skeleton_condition against the reference's own class (live where the
reference tree is installed, through the golden vectors of oracle/make_golden_skeleton.py everywhere), its float32
rounding against float64, and the mirror's refusal of CPU tensors."""
import os

import numpy as np
import pytest
import torch

from oracle import ref_loader as RL
from oracle.skeleton_condition import mdm_skeleton_condition
from tests.helpers import rel
from tests.skeleton_helpers import GOLDEN_CASES, mirror_args, skeleton_encoder_weights, skeleton_inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_ref = pytest.mark.skipif(not RL.available(), reason="reference tree not present")


def _condition(sd, B, T, P, faithful=False):
    body, obj, pose, zp = skeleton_inputs(B, T, P)
    with torch.no_grad():
        return mdm_skeleton_condition(sd, body, obj, zp, P, faithful=faithful)


@needs_ref
@pytest.mark.parametrize("faithful", [True, False])
@pytest.mark.parametrize("B,T,P", [(3, 15, 10), (2, 30, 17), (2, 8, 10)])
def test_restatement_matches_reference_class(faithful, B, T, P):
    """the shipped checkpoint through the reference's own MDM._get_embeddings vs the restatement, same inputs"""
    model, _, _ = RL.build_mdm_skeleton(diffusion_steps=1000, past_len=P)
    _, sd = RL.load_ckpt("diffusion_skeleton")
    body, obj, pose, zp = skeleton_inputs(B, T, P)
    with torch.no_grad():
        ref, gt = model._get_embeddings(body, obj, pose, zp)
        got = mdm_skeleton_condition(sd, body, obj, zp, P, faithful=faithful)
    assert got.shape == (min(P, T), B, 256)
    assert rel(got, ref) < 1e-5


@pytest.mark.parametrize("source", ["random", "ref"])
def test_restatement_matches_golden(source):
    """against tests/golden/skeleton_condition_<source>.npz (the reference class's outputs on the same weights and inputs)"""
    sd = skeleton_encoder_weights(source)
    with np.load(os.path.join(GOLDEN, "skeleton_condition_%s.npz" % source)) as g:
        for B, T, P in GOLDEN_CASES:
            key = "%d_%d_%d" % (B, T, P)
            want = torch.from_numpy(g["cond_" + key])
            assert want.shape == (min(P, T), B, 256)
            for faithful in (True, False):
                assert rel(_condition(sd, B, T, P, faithful), want) < 1e-5, (key, faithful)
            body, obj, pose, _ = skeleton_inputs(B, T, P)
            assert torch.equal(torch.cat([body.reshape(T, B, -1), obj.reshape(T, B, -1), pose], dim=2), torch.from_numpy(g["gt_" + key]))


@pytest.mark.parametrize("source", ["random", "ref"])
def test_float32_rounding_spread(source, record_property):
    """the float32 restatement against the same computation in float64: the rounding the device's 2e-4 bound has to absorb"""
    sd = skeleton_encoder_weights(source)
    sd64 = {k: v.double() for k, v in sd.items()}
    spread = {}
    for B, T, P in GOLDEN_CASES:
        body, obj, _, zp = skeleton_inputs(B, T, P)
        with torch.no_grad():
            f32 = mdm_skeleton_condition(sd, body, obj, zp, P, faithful=False)
            f64 = mdm_skeleton_condition(sd64, body.double(), obj.double(), zp.double(), P, faithful=False)
        spread["%d_%d_%d" % (B, T, P)] = rel(f32, f64)
    record_property("float32_vs_float64", spread)
    assert max(spread.values()) < 2e-5, spread


def test_mirror_refuses_cpu_tensors():
    from interdiff_b200.model.diffusion_skeleton import MDM
    model = MDM(mirror_args())
    body, obj, pose, zp = skeleton_inputs(2, 15, 10)
    with pytest.raises(RuntimeError, match="CUDA"):
        model._get_embeddings(body, obj, pose, zp)
