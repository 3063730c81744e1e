"""Pins oracle.restate against the reference's OWN classes (imported through oracle.shims) with the shipped checkpoints.
The tests that need the checkpoints run only where the reference tree is installed; elsewhere the golden-vector tests
(tests/test_golden.py: the same classes on seeded weights) take over.  The SMPL-H layer and the `smooth` comparison need no
checkpoint: they always compare with the reference's stored outputs (tests/golden/smplh_lbs.npz, smooth.npz, written by
oracle/make_golden.py) and, where the tree is installed, check those stored outputs against a live run as well."""
import ast
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

from interdiff_b200 import synthetic as S
from oracle import ref_loader as RL
from oracle import restate as R
from oracle import transforms as tf

needs_ref = pytest.mark.skipif(not RL.available(), reason="reference tree not present")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, b):
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


@pytest.fixture(scope="module")
def mdm():
    model, diffusion, args = RL.build_mdm_smpl(diffusion_steps=1000)
    _, sd = RL.load_ckpt("diffusion")
    return model, diffusion, args, sd


def _kw(b):
    return {"y": {"cond": torch.from_numpy(b["cond"]), "inpainted_motion": torch.from_numpy(b["gt"]),
                  "inpainting_mask": torch.from_numpy(b["mask"])}}


@pytest.mark.parametrize("rotary", ["absolute", "bucketed"])
@pytest.mark.parametrize("faithful", [True, False])
@needs_ref
def test_mdm_forward(mdm, rotary, faithful):
    model, _, _, sd = mdm
    for m in model.modules():
        if hasattr(m, "rotary"):
            m.rotary = rotary
    b = S.make_smpl_batch(B=3, T=30)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([999, 500, 0])
    with torch.no_grad():
        ref = model(x, t, y={"cond": torch.from_numpy(b["cond"])})
        got = R.mdm_smpl_forward(sd, x, t, torch.from_numpy(b["cond"]), rotary=rotary, faithful=faithful)
    for m in model.modules():
        if hasattr(m, "rotary"):
            m.rotary = "absolute"
    assert rel(got, ref) < 2e-5


@pytest.mark.parametrize("faithful", [True, False])
@needs_ref
def test_condition_encoder(mdm, faithful):
    """oracle.mdm_smpl_condition against the reference's own modules on the same inputs: bodyEmbedding /
    objEmbedding of the past frames + point-cloud embedding, PositionalEmbedding, encoder
    (model/diffusion_smpl.py:217-221)."""
    model, _, args, sd = mdm
    B, T = 3, 30
    b = S.make_smpl_batch(B=B, T=T)
    gt = torch.from_numpy(b["gt"])
    past = gt[..., : args.past_len].contiguous()
    pc = torch.randn(B, 256, generator=torch.Generator().manual_seed(4))
    xs = past.squeeze(1).permute(2, 0, 1)
    with torch.no_grad():
        emb = model.bodyEmbedding(xs[..., :135]) + model.objEmbedding(xs[..., 135:]) + pc[None]
        ref = model.encoder(model.PositionalEmbedding(emb))
        got = R.mdm_smpl_condition(sd, past, pc, faithful=faithful)
    assert rel(got, ref) < 2e-5


@needs_ref
def test_p_sample_loop_short(mdm):
    model, _, args, sd = mdm
    steps = 6
    m = RL.modules()["model.diffusion_smpl"]
    a = Namespace(**{**vars(args), "diffusion_steps": steps})
    diffusion = m.create_gaussian_diffusion(a)
    b = S.make_smpl_batch(B=2, T=30)
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps))
    gd = RL.modules()["diffusion.gaussian_diffusion"]
    idx = [0]

    def fake(x):
        idx[0] += 1
        return tape[idx[0]].clone()
    old, gd.th.randn_like = gd.th.randn_like, fake
    try:
        with torch.no_grad():
            ref = diffusion.p_sample_loop(model, b["gt"].shape, noise=tape[0].clone(), clip_denoised=False,
                                          model_kwargs=_kw(b))
    finally:
        gd.th.randn_like = old
    tables = R.diffusion_tables(R.named_beta_schedule("cosine", steps))
    for k in ("posterior_mean_coef1", "posterior_mean_coef2", "posterior_log_variance_clipped"):
        assert np.array_equal(tables[k], getattr(diffusion, k))
    cond = torch.from_numpy(b["cond"])
    with torch.no_grad():
        got = R.p_sample_loop(lambda x, t: R.mdm_smpl_forward(sd, x, t, cond), tables, tape,
                              gt=torch.from_numpy(b["gt"]), mask=torch.from_numpy(b["mask"]))
    assert rel(got, ref) < 1e-3  # a 6-step chain ends on the ill-conditioned t=1,0 steps (DESIGN.md "Conditioning")


@needs_ref
def test_skeleton_forward():
    model, diffusion, args = RL.build_mdm_skeleton(diffusion_steps=1000)
    _, sd = RL.load_ckpt("diffusion_skeleton")
    b = S.make_skeleton_batch(B=2, T=15)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([999, 3])
    zp = torch.from_numpy(b["zero_pose_obj"])
    with torch.no_grad():
        ref = model(x, t, zp, y={"cond": torch.from_numpy(b["cond"])})
        got = R.mdm_skeleton_forward(sd, x, t, zp, torch.from_numpy(b["cond"]))
    assert rel(got, ref) < 2e-5


def test_smplh_lbs(smplh_np):
    from oracle import make_golden as MG
    smplh = {k: torch.from_numpy(np.asarray(v)) for k, v in smplh_np.items()}
    pose, betas, trans = MG.lbs_inputs()
    gold = np.load(os.path.join(GOLDEN, "smplh_lbs.npz"))
    v_ref, j_ref = torch.from_numpy(gold["verts"]), torch.from_numpy(gold["jtr"])
    with torch.no_grad():
        v, j = R.smplh_lbs(smplh, pose, betas, trans)
    assert rel(v[:, ::MG.LBS_VERTEX_STRIDE], v_ref) < 1e-6 and rel(j, j_ref) < 1e-6
    if RL.available():      # the stored vectors are what the reference's layer computes, and the unsampled vertices agree too
        v_live, j_live = MG.reference_lbs(smplh_np)
        assert torch.equal(v_live[:, ::MG.LBS_VERTEX_STRIDE], v_ref) and torch.equal(j_live, j_ref)
        assert rel(v, v_live) < 1e-6


@needs_ref
def test_geometry_helpers(smplh_np):
    mods = RL.modules()
    g = torch.Generator().manual_seed(2)
    verts = torch.from_numpy(smplh_np["v_template"])[None].repeat(2, 1, 1) + 0.01 * torch.randn(2, 6890, 3, generator=g)
    faces = torch.from_numpy(smplh_np["faces"])
    n_ref = mods["data.tools"].vertex_normals(verts, faces.unsqueeze(0).repeat(2, 1, 1))
    n = R.vertex_normals(verts, faces)
    assert rel(n, n_ref) < 1e-5
    y = 0.3 * torch.randn(2, 300, 3, generator=g)
    ref = mods["tools"].point2point_signed(verts, y, x_normals=n_ref, return_vector=True)
    got = R.point2point_signed(verts, y, n_ref)
    assert torch.equal(got[2].long(), ref[2].long()) and torch.equal(got[3].long(), ref[3].long())
    assert rel(got[0], ref[0]) < 1e-6 and rel(got[1], ref[1]) < 1e-6


@needs_ref
def test_obj_projector():
    model, args = RL.build_obj_projector(past_len=10, future_len=20)
    _, sd = RL.load_ckpt("correction")
    g = torch.Generator().manual_seed(3)
    T, B = 30, 5
    ang = torch.randn(T, B, 6, generator=g)
    tr = torch.randn(T, B, 3, generator=g)
    hv = torch.randn(T, B, 67, 3, generator=g)
    contact = (torch.rand(B, 67, generator=g) < 0.05).long() * torch.randint(1, 5, (B, 67), generator=g)
    contact[1] = 0
    with torch.no_grad():
        ref = model.sample(ang, tr, hv, contact)
        got = R.obj_projector_sample(sd, ang, tr, hv, contact, 10, 20)
    assert rel(got, ref) < 1e-5


@needs_ref
def test_obj_projector_skeleton():
    """oracle restatement of the skeleton correction net against the reference class with checkpoints/obj_skeleton.ckpt
    (SURVEY 8f rank 4: the CUDA side of this row is not built yet; this pins the checker for it)."""
    model, args, sd = RL.build_obj_projector_skeleton()
    g = torch.Generator().manual_seed(8)
    T, B = args.past_len + args.future_len, 4
    quat = torch.nn.functional.normalize(torch.randn(T, B, 4, generator=g), dim=2)
    tr = torch.randn(T, B, 3, generator=g)
    hp = torch.randn(T, B, args.num_joints, 3, generator=g)
    with torch.no_grad():
        ref_q, ref_t = model.sample(quat, tr, hp)
        got_q, got_t = R.obj_projector_skeleton_sample(sd, quat, tr, hp, args.past_len, args.future_len)
    assert rel(got_q, ref_q) < 1e-5 and rel(got_t, ref_t) < 1e-5


def _reference_function(fname, name, env):
    """Compile ONE function of a reference script (the script itself cannot be imported: it
    pulls pytorch_lightning / psbody / render at module level) into `env`."""
    path = os.path.join(RL.ref_root(), "interdiff", fname)
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name][0]
    code = compile(ast.Module(body=[fn], type_ignores=[]), path, "exec")
    exec(code, env)
    return env[name]


@needs_ref
def test_metrics(smplh_np):
    """oracle.metrics against the reference's own `metrics` function (eval_smpl_short.py:24-81) compiled out of the
    script, with the script's imports bound to the reference's tools / data.tools and the transforms shim."""
    mods = RL.modules()
    env = {"torch": torch, "axis_angle_to_matrix": tf.axis_angle_to_matrix, "axis_angle_to_quaternion": tf.axis_angle_to_quaternion,
           "vertex_normals": mods["data.tools"].vertex_normals, "point2point_signed": mods["tools"].point2point_signed}
    ref_fn = _reference_function("eval_smpl_short.py", "metrics", env)
    from tests.helpers import metrics_inputs
    a = metrics_inputs(smplh_np)
    with torch.no_grad():
        ref = ref_fn(**a)
        got = R.metrics(**a)
    for k in ref:
        assert rel(got[k], ref[k]) < 1e-5, k
    assert float(ref["penetrate"].max()) > 0            # the batch does exercise penetration


def test_smooth_and_best_of_samples():
    """host-side post-processing mirrors (interdiff_b200.sampling.smooth / BestOfSamples) against the reference's
    `smooth` (eval_smpl_short.py:217-223) and the min-over-draws reduction of its evaluation loop (:268-296)."""
    from interdiff_b200 import sampling
    from oracle import make_golden as MG
    g, xs = MG.smooth_inputs()
    gold = np.load(os.path.join(GOLDEN, "smooth.npz"))
    ref = [torch.from_numpy(gold["out%d" % i]) for i in range(len(xs))]
    got = sampling.smooth(*[x.clone() for x in xs], future_len=20)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    if RL.available():
        for a, b in zip(MG.reference_smooth(), ref):
            assert torch.equal(a, b)
    acc = sampling.BestOfSamples(names=("m",))
    draws = [torch.rand(4, generator=g) for _ in range(3)]
    acc.start_batch()
    for d in draws:
        acc.add({"m": d})
    acc.end_batch()
    want = torch.stack([torch.full((4,), 1e10)] + draws).min(dim=0)[0].mean().item()
    assert abs(acc.averages()["m"] - want) < 1e-7


@needs_ref
def test_denoised_fn(smplh_np):
    """oracle.restate.make_denoised_fn against the reference's own denoised_fn source
    (eval_smpl_short.py:84-130) executed with the reference's ObjProjector / SMPL_Layer /
    vertex_normals / point2point_signed."""
    mods = RL.modules()
    T, B = 30, 2
    b = S.make_smpl_batch(B=B, T=T)
    layer = RL.build_smpl_layer(smplh_np)
    proj, pargs = RL.build_obj_projector(past_len=10, future_len=20)
    _, psd = RL.load_ckpt("correction")
    args = Namespace(smpl_dim=132, past_len=10, future_len=20)
    env = dict(torch=torch, args=args, rotation_6d_to_matrix=tf.rotation_6d_to_matrix,
               matrix_to_axis_angle=tf.matrix_to_axis_angle,
               markerset_ssm67_smplh=mods["data.utils"].markerset_ssm67_smplh,
               vertex_normals=mods["data.tools"].vertex_normals,
               point2point_signed=mods["tools"].point2point_signed)
    ref_fn = _reference_function("eval_smpl_short.py", "denoised_fn", env)
    gt = torch.from_numpy(b["gt"])
    # a prediction near the ground truth (so contacts / penetration decisions are exercised)
    g = torch.Generator().manual_seed(4)
    x = gt + 0.02 * torch.randn(gt.shape, generator=g)
    kw = {"y": {"inpainted_motion": gt, "hand_pose": torch.from_numpy(b["hand_pose"]), "smpl": layer,
                "beta": torch.from_numpy(b["betas"]), "obj_model": Namespace(model=proj),
                "obj_points": torch.from_numpy(b["obj_points"])}}
    smplh = {k: torch.from_numpy(np.asarray(v)) for k, v in smplh_np.items()}
    ctx = dict(past_len=10, future_len=20, smpl_dim=132, gt=gt, hand_pose=kw["y"]["hand_pose"],
               betas=kw["y"]["beta"], obj_points=kw["y"]["obj_points"], smplh=smplh, projector=psd)
    fn = R.make_denoised_fn(ctx)
    for tval in (450, 0, 7):
        t = torch.full((B,), tval, dtype=torch.long)
        with torch.no_grad():
            ref = ref_fn(x.clone(), t, kw)
            got = fn(x.clone(), t, None)
        assert rel(got, ref) < 1e-5, tval
    obs = R.correction_observables(x, ctx)
    assert obs["condition"].shape == (B,)
