"""The skeleton model's conditioning encoder on the device (idb_encode_condition_skeleton: reference
model/diffusion_skeleton.py:194-215) against oracle.skeleton_condition, and the skeleton drivers it unlocks replayed
through the mirrored modules: eval_skeleton.py's sample_once_proj (:114-142) with the plain-Python hook and with
sampling.FusedSkeletonCorrection, and the validation branch of train_diffusion_skeleton.py (:255-283).
Tolerances: max|a-b| / max|b|."""
import ctypes as C
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

from interdiff_b200 import synthetic as S
from oracle import restate as R
from oracle import transforms as tf
from oracle.skeleton_condition import mdm_skeleton_condition
from tests.helpers import encoder_weights, mdm_weights, projector_skeleton_weights, rel
from tests.skeleton_helpers import GOLDEN_CASES, mirror_args, skeleton_encoder_weights, skeleton_inputs

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", params=["simt", "tcgen05"])
def eng(request):
    from interdiff_b200.engine import Engine
    e = Engine("cuda:0")
    e.set_gemm_backend(request.param)
    yield e
    e.close()


_SD = {}


def _weights(source):
    if source not in _SD:
        _SD[source] = skeleton_encoder_weights(source)
    return _SD[source]


def _encode(eng, B, T, Tp):
    body, obj, _, zp = skeleton_inputs(B, T)
    return eng.encode_condition_skeleton(body.cuda(), obj.cuda(), zp.cuda(), Tp), (body, obj, zp)


@pytest.mark.parametrize("source", ["random", "ref"])
@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("Tp", [1, 10, 17, 36])
def test_condition_vs_oracle_then_forward(eng, source, B, Tp):
    """cond at 2e-4 of the oracle (Tp > 16: two attention slabs per sample; the inputs are transposed views, as the
    evaluation script passes them), then bind + forward on it at 3e-4 of the oracle's forward on the oracle's cond"""
    sd = _weights(source)
    eng.load_denoiser(sd, "skeleton")
    cond, (body, obj, zp) = _encode(eng, B, Tp + 3, Tp)
    with torch.no_grad():
        ref = mdm_skeleton_condition(sd, body, obj, zp, Tp, faithful=False)
    assert cond.shape == (Tp, B, 256)
    assert rel(cond, ref) < 2e-4
    Tm, T = min(Tp, 16), 15
    eng.bind(cond[:Tm], T, zero_pose_obj=zp)
    x = torch.from_numpy(S.noise_tape((B, 1, 106, T), 0, seed=B)[0])
    t = torch.arange(B) * 997 % 1000
    got = eng.forward(x.cuda(), t.cuda()).cpu()
    with torch.no_grad():
        want = R.mdm_skeleton_forward(sd, x, t, zp, ref[:Tm], faithful=False)
    assert rel(got, want) < 3e-4


@pytest.mark.parametrize("source", ["random", "ref"])
def test_condition_vs_golden(eng, source):
    """against the reference class's own outputs stored by oracle/make_golden_skeleton.py"""
    sd = _weights(source)
    eng.load_denoiser(sd, "skeleton")
    with np.load(os.path.join(GOLDEN, "skeleton_condition_%s.npz" % source)) as g:
        for B, T, P in GOLDEN_CASES:
            cond, _ = _encode(eng, B, T, min(P, T))
            assert rel(cond, torch.from_numpy(g["cond_%d_%d_%d" % (B, T, P)])) < 2e-4, (B, T, P)


def test_bits_independent_of_launch_mode_and_batch(eng):
    """the same bits with programmatic dependent launch on and off, and for a slice of the batch (M = 8*17 rows) as
    for the full batch (M = 64*17)"""
    eng.load_denoiser(_weights("random"), "skeleton")
    B, T, Tp = 64, 20, 17
    full, (body, obj, zp) = _encode(eng, B, T, Tp)
    full = full.clone()
    eng.set_dependent_launch(False)
    try:
        off, _ = _encode(eng, B, T, Tp)
    finally:
        eng.set_dependent_launch(True)
    assert torch.equal(off, full)
    sl = slice(24, 32)
    part = eng.encode_condition_skeleton(body[:, sl].cuda(), obj[:, sl].cuda(), zp[sl].cuda(), Tp)
    assert torch.equal(part, full[:, sl])


def test_argument_rejection():
    """status codes of the C entry points: 2 = argument, 3 = state"""
    from interdiff_b200.engine import Engine
    e = Engine("cuda:0")
    B, Tp = 2, 37
    body, obj, zp = torch.zeros(Tp, B, 21, 3).cuda(), torch.zeros(Tp, B, 12, 3).cuda(), torch.zeros(B, 12, 3).cuda()
    out = torch.empty(Tp, B, 256, device="cuda")
    pc = torch.zeros(B, 256, device="cuda")
    P = lambda t: C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    skel = lambda tp, b=B, o=out: e.lib.idb_encode_condition_skeleton(e._h, b, tp, P(body), P(obj), P(zp), P(o), st)
    try:
        e.load_denoiser(_weights("random"), "skeleton")
        assert skel(10) == 0
        assert skel(37) == 2 and skel(0) == 2 and skel(10, b=0) == 2
        assert e.lib.idb_encode_condition_skeleton(e._h, B, 10, P(body), C.c_void_p(), P(zp), P(out), st) == 2
        with pytest.raises(Exception, match="36 frames"):
            e.encode_condition_skeleton(body, obj, zp, 37)
        # a skeleton handle through the SMPL entry point
        past = torch.zeros(B, 1, 144, 10, device="cuda")
        assert e.lib.idb_encode_condition(e._h, B, 10, P(past), P(pc), P(out), st) == 2
        # the skeleton weights without shapeEmbedding.*
        e.load_denoiser({k: v for k, v in _weights("random").items() if not k.startswith("shapeEmbedding.")}, "skeleton")
        assert skel(10) == 3 and "shapeEmbedding" in e.lib.idb_last_error(e._h).decode()
        # an SMPL handle
        e.load_denoiser(encoder_weights("random"), "smpl")
        assert skel(10) == 2
        torch.cuda.synchronize()
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# the skeleton drivers through the mirrored modules
# ------------------------------------------------------------------------------------------------------------------
class _ObjModel:            # the script passes the Lightning module; the hook reads `.model` (eval_skeleton.py:101)
    def __init__(self, m):
        self.model = m


def _mirror(steps, P=10, Fu=10):
    from interdiff_b200.model.correction_skeleton import ObjProjector
    from interdiff_b200.model.diffusion_skeleton import create_model_and_diffusion
    model, diffusion = create_model_and_diffusion(mirror_args(diffusion_steps=steps, past_len=P, future_len=Fu))
    sd = _weights("random")
    own = model.state_dict()
    model.load_state_dict({k: (sd[k].reshape(own[k].shape) if k in sd else v) for k, v in own.items()})
    proj = ObjProjector(Namespace(num_joints=21, dropout=0.0, past_len=P, future_len=Fu, embedding_dim=128))
    psd = projector_skeleton_weights("random")
    own = proj.state_dict()
    proj.load_state_dict({k: (psd[k].reshape(own[k].shape) if k in psd else v) for k, v in own.items()}, strict=True)
    return model.cuda().eval(), diffusion, {k: v.cpu() for k, v in model.state_dict().items()}, proj.cuda().eval(), psd


def _script_denoised_fn():
    """eval_skeleton.py:80-111 transcribed onto the mirrored modules (calc_obj_pred :34-44 with oracle.transforms'
    pure-torch quaternion_to_matrix, which runs on CUDA tensors like any torch code)"""
    def calc_obj_pred(pose_pred, zero_pose_obj):
        quat_correct = torch.cat([pose_pred[:, :, -1, None], pose_pred[:, :, -4:-1]], dim=2)
        rotation_matrix = tf.quaternion_to_matrix(quat_correct)[:, :, None]
        return (rotation_matrix.matmul(zero_pose_obj[None, :, :, :, None]) + pose_pred[:, :, None, :3, None])[:, :, :, :, 0]

    def denoised_fn(x, t, model_kwargs):
        if t[0] > 500 or t[0] % 50 != 0:
            return x
        body_pred, obj_pred, _ = torch.split(x.squeeze(1).permute(2, 0, 1).contiguous(), [21 * 3, 12 * 3, 7], dim=2)
        _, obj_gt, pose_gt = torch.split(model_kwargs["y"]["inpainted_motion"].squeeze(1).permute(2, 0, 1).contiguous(), [21 * 3, 12 * 3, 7], dim=2)
        T, B, _ = body_pred[:, :, :-3].shape
        obj_trans_gt, obj_angles_gt = torch.split(pose_gt, [3, 4], dim=2)
        obj_model = model_kwargs["y"]["obj_model"]
        obj_angles_proj, obj_trans_proj = obj_model.model.sample(obj_angles_gt, obj_trans_gt, body_pred.view(T, B, -1, 3))
        pose_proj = torch.cat([obj_trans_proj, obj_angles_proj], dim=2)
        obj_proj = calc_obj_pred(pose_proj, model_kwargs["zero_pose_obj"]).view(T, B, -1)
        x_ = torch.cat([body_pred, obj_proj, pose_proj], dim=2).permute(1, 2, 0).unsqueeze(1).contiguous()
        denoised_fn.calls += 1
        return t[0] / 1000 * x + (1 - t[0] / 1000) * x_
    denoised_fn.calls = 0
    return denoised_fn


def test_eval_skeleton_sample_once_proj():
    """eval_skeleton.py:114-142 through the mirrored API only, 52-step schedule (hook active at i = 50 and i = 0), seeded
    random-init weights (a well-conditioned chain, as in test_gpu_configs.py::test_skeleton_correction):
      embedding, gt = model._get_embeddings(body_gt, obj_gt, pose_gt, zero_pose_obj) -> p_sample_loop(..., denoised_fn).
    The fused hook object equals Engine.p_sample_loop(correction=True) on the same cond and tape bit for bit; the
    script's plain hook (step by step) agrees with it, and both with the oracle chain, at 1e-3."""
    from interdiff_b200.sampling import FusedSkeletonCorrection, draw_tape
    steps, B, P, Fu = 52, 4, 10, 10
    T = P + Fu
    model, diffusion, msd, proj, psd = _mirror(steps, P, Fu)
    body_gt, obj_gt, pose_gt, zp = (x.cuda() for x in skeleton_inputs(B, T, P))      # transposed views, as the script has them
    with torch.no_grad():
        embedding, gt = model._get_embeddings(body_gt, obj_gt, pose_gt, zp)
    assert embedding.shape == (P, B, 256) and gt.shape == (T, B, 106)
    gt = gt.permute(1, 2, 0).unsqueeze(1).contiguous()
    mask = torch.ones_like(gt, dtype=torch.bool)
    mask[:, :, :, P:] = False
    kw = lambda: {"y": {"cond": embedding, "inpainted_motion": gt, "inpainting_mask": mask, "obj_model": _ObjModel(proj)}, "zero_pose_obj": zp}
    noise = torch.randn(gt.shape, generator=torch.Generator().manual_seed(3)).cuda()
    torch.manual_seed(11)
    fused = diffusion.p_sample_loop(model, gt.shape, clip_denoised=False, noise=noise, model_kwargs=kw(),
                                    denoised_fn=FusedSkeletonCorrection()).clone()
    eng = model.engine_for(gt.device)
    torch.manual_seed(11)
    tape = draw_tape(eng, noise, steps)
    direct = eng.p_sample_loop(tape, gt, mask, correction=True).clone()
    assert torch.equal(fused, direct)
    fn = _script_denoised_fn()
    torch.manual_seed(11)
    py = diffusion.p_sample_loop(model, gt.shape, clip_denoised=False, noise=noise, model_kwargs=kw(), denoised_fn=fn)
    assert fn.calls == 2
    assert rel(py, fused) < 1e-3
    # the oracle chain: oracle cond -> oracle sampling loop with the restated hook, same tape
    gtc, zpc = gt.cpu(), zp.cpu()
    with torch.no_grad():
        cond_ref = mdm_skeleton_condition(msd, body_gt.cpu(), obj_gt.cpu(), zpc, P, faithful=False)
        ctx = dict(gt=gtc, zero_pose_obj=zpc, projector=psd, past_len=P, future_len=Fu)
        tables = R.diffusion_tables(R.named_beta_schedule("cosine", steps))
        fwd = lambda x, t: R.mdm_skeleton_forward(msd, x, t, zpc, cond_ref, faithful=False)
        ref = R.p_sample_loop(fwd, tables, tape.cpu(), gtc, mask.cpu(), denoised_fn=R.make_denoised_fn_skeleton(ctx))
        plain = R.p_sample_loop(fwd, tables, tape.cpu(), gtc, mask.cpu())
    assert rel(fused, ref) < 1e-3 and rel(py, ref) < 1e-3
    assert rel(plain, ref) > 1e-3            # the hook changed the sample: the comparisons above are not vacuous
    # the fused hook object called directly (as a plain callback) is the same gate + kernels
    x0 = direct.clone()
    hook = FusedSkeletonCorrection()
    assert hook(x0, torch.full((B,), 51, device="cuda"), kw()) is x0 and torch.equal(x0, direct)
    want = eng.skeleton_correction_apply(direct.clone(), gt, zp, 450)
    assert torch.equal(hook(direct.clone(), torch.full((B,), 450, device="cuda"), kw()), want)


def test_train_skeleton_valid_branch_is_one_loop_call():
    """train_diffusion_skeleton.py:255-283 (mode 'valid'): _get_embeddings, then p_sample_loop(model, gt.shape,
    clip_denoised=False, model_kwargs) without noise or hook: one library loop call, equal to the Engine loop on the
    same x_T and tape"""
    from interdiff_b200.sampling import draw_tape
    steps, B, P, T = 8, 3, 10, 25
    model, diffusion, _, _, _ = _mirror(steps, P, T - P)
    batch = skeleton_inputs(B, T, P)
    body_gt, obj_gt, pose_gt = (x.float().cuda() for x in batch[:3])
    zero_pose_obj = batch[3].float().cuda()
    with torch.no_grad():
        embedding, gt = model._get_embeddings(body_gt, obj_gt, pose_gt, zero_pose_obj)
    gt = gt.permute(1, 2, 0).unsqueeze(1).contiguous()
    model_kwargs = {"y": {"cond": embedding}, "zero_pose_obj": zero_pose_obj}
    model_kwargs["y"]["inpainted_motion"] = gt
    model_kwargs["y"]["inpainting_mask"] = torch.ones_like(gt, dtype=torch.bool, device="cuda")
    model_kwargs["y"]["inpainting_mask"][:, :, :, P:] = False
    eng = model.engine_for(gt.device)
    calls, orig = [], eng.p_sample_loop
    eng.p_sample_loop = lambda *a, **k: calls.append(1) or orig(*a, **k)
    try:
        torch.manual_seed(5)
        sample = diffusion.p_sample_loop(model, gt.shape, clip_denoised=False, model_kwargs=model_kwargs).clone()
    finally:
        del eng.p_sample_loop
    assert calls == [1]
    mask = model_kwargs["y"]["inpainting_mask"]
    torch.manual_seed(5)
    x_T = torch.randn(*gt.shape, device="cuda")
    x_T = (x_T * ~mask) + (gt * mask)
    tape = draw_tape(eng, x_T, steps)
    assert torch.equal(sample, eng.p_sample_loop(tape, gt, mask))
    assert torch.equal(sample[..., :P], gt[..., :P]) and torch.isfinite(sample).all()
