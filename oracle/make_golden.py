"""Generate tests/golden/*.npz from the reference's OWN classes (imported via
oracle.shims) -- run where the reference tree is installed:  python -m oracle.make_golden
TEST INFRASTRUCTURE.  Inputs are the seeded synthetic generators of interdiff_b200.synthetic;
weights are either the seeded random init (portable: regenerated from the seed by the tests) or
the shipped checkpoints (tests using those need oracle/_ref/weights, else skip).
"""
import ast
import os
import sys
from argparse import Namespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from interdiff_b200 import synthetic as S  # noqa: E402
from oracle import ref_loader as RL  # noqa: E402
from oracle import transforms as tf  # noqa: E402
from tests.helpers import encoder_weights, mdm_weights, projector_weights  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def run_loop(diffusion, model, tape, kw, extra=None, denoised_fn=None):
    gd = RL.modules()["diffusion.gaussian_diffusion"]
    idx = [0]

    def fake(x):
        idx[0] += 1
        return tape[idx[0]].clone()
    old, gd.th.randn_like = gd.th.randn_like, fake
    try:
        with torch.no_grad():
            mk = dict(kw)
            if extra:
                mk.update(extra)
            return diffusion.p_sample_loop(model, tuple(tape[0].shape), noise=tape[0].clone(), clip_denoised=False,
                                           model_kwargs=mk, denoised_fn=denoised_fn)
    finally:
        gd.th.randn_like = old


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    for source in ("random", "ref"):
        # ---- SMPL denoiser forward + 5-step loop
        sd = mdm_weights("smpl", source)
        model, _, args = RL.build_mdm_smpl(state_dict=sd, diffusion_steps=1000)
        b = S.make_smpl_batch(B=2, T=30)
        x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
        t = torch.tensor([999, 3])
        cond = torch.from_numpy(b["cond"])
        with torch.no_grad():
            out = model(x, t, y={"cond": cond})
        steps = 5
        a = Namespace(**{**vars(args), "diffusion_steps": steps})
        diffusion = RL.modules()["model.diffusion_smpl"].create_gaussian_diffusion(a)
        tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps))
        kw = {"y": {"cond": cond, "inpainted_motion": torch.from_numpy(b["gt"]), "inpainting_mask": torch.from_numpy(b["mask"])}}
        loop = run_loop(diffusion, model, tape, kw)
        np.savez_compressed(os.path.join(OUT, "mdm_smpl_%s.npz" % source), forward=out.numpy(), t=t.numpy(), loop5=loop.numpy())
        # ---- conditioning encoder (the part of MDM._get_embeddings after the point-cloud encoder)
        esd = encoder_weights(source)
        emodel, _, eargs = RL.build_mdm_smpl(state_dict=esd, diffusion_steps=1000)
        past = torch.from_numpy(b["gt"])[..., : eargs.past_len].contiguous()
        pc = torch.randn(2, 256, generator=torch.Generator().manual_seed(7))
        xs = past.squeeze(1).permute(2, 0, 1)
        with torch.no_grad():
            emb = emodel.bodyEmbedding(xs[..., :135]) + emodel.objEmbedding(xs[..., 135:]) + pc[None]
            cond_out = emodel.encoder(emodel.PositionalEmbedding(emb))
        # point-cloud encoder: the reference's own PointNet2Encoder class on the restated pointnet2_ops operators
        op = torch.from_numpy(b["obj_points"])
        with torch.no_grad():
            pc_pts = emodel.pcEmbedding(torch.cat([op, op.norm(dim=2, keepdim=True)], dim=2).unsqueeze(0)).view(1, 2, -1)[0]
        np.savez_compressed(os.path.join(OUT, "cond_encoder_%s.npz" % source), pc=pc.numpy(), cond=cond_out.numpy(),
                            pc_from_points=pc_pts.numpy())
        # ---- skeleton denoiser, BASELINE config 1: 1 DDPM step, B=2, T=15
        sd = mdm_weights("skeleton", source)
        model, _, args = RL.build_mdm_skeleton(state_dict=sd, diffusion_steps=1000)
        b = S.make_skeleton_batch(B=2, T=15)
        x = torch.from_numpy(S.noise_tape(b["gt"].shape, 1)[0])
        zp = torch.from_numpy(b["zero_pose_obj"])
        with torch.no_grad():
            out = model(x, torch.tensor([999, 999]), zp, y={"cond": torch.from_numpy(b["cond"])})
        a = Namespace(**{**vars(args), "diffusion_steps": 1})
        # a 1-step schedule has posterior_variance[1] undefined in the reference; use the 1000-step
        # process and execute ONE p_sample at t=999 (config 1: "1 DDPM step")
        diffusion = RL.modules()["model.diffusion_skeleton"].create_gaussian_diffusion(Namespace(**{**vars(args), "diffusion_steps": 1000}))
        tape = torch.from_numpy(S.noise_tape(b["gt"].shape, 1))
        kw = {"y": {"cond": torch.from_numpy(b["cond"]), "inpainted_motion": torch.from_numpy(b["gt"]),
                    "inpainting_mask": torch.from_numpy(b["mask"])}, "zero_pose_obj": zp}
        gd = RL.modules()["diffusion.gaussian_diffusion"]
        old, gd.th.randn_like = gd.th.randn_like, (lambda x_: tape[1].clone())
        try:
            with torch.no_grad():
                st = diffusion.p_sample(model, tape[0].clone(), torch.tensor([999, 999]), clip_denoised=False, model_kwargs=kw)
        finally:
            gd.th.randn_like = old
        np.savez_compressed(os.path.join(OUT, "mdm_skeleton_%s.npz" % source), forward=out.numpy(), step_sample=st["sample"].numpy(),
                            step_x0=st["pred_xstart"].numpy())
        # ---- projector
        psd = projector_weights(source)
        proj, _ = RL.build_obj_projector(state_dict=psd, past_len=10, future_len=20)
        g = torch.Generator().manual_seed(3)
        T, B = 30, 4
        ang, tr, hv = torch.randn(T, B, 6, generator=g), torch.randn(T, B, 3, generator=g), torch.randn(T, B, 67, 3, generator=g)
        contact = (torch.rand(B, 67, generator=g) < 0.05).long() * torch.randint(1, 5, (B, 67), generator=g)
        contact[1] = 0
        with torch.no_grad():
            pout = proj.sample(ang, tr, hv, contact)
        np.savez_compressed(os.path.join(OUT, "projector_%s.npz" % source), ang=ang.numpy(), tr=tr.numpy(), hv=hv.numpy(),
                            contact=contact.numpy(), out=pout.numpy())

    # ---- geometry: LBS, normals, signed NN (synthetic SMPL-H, no learned weights)
    smplh = S.make_smplh_model(233)
    layer = RL.build_smpl_layer(smplh)
    g = torch.Generator().manual_seed(1)
    Fn = 5
    pose = 0.4 * torch.randn(Fn, 156, generator=g)
    pose[0, 3:6] = 0
    betas, trans = torch.randn(Fn, 10, generator=g), torch.randn(Fn, 3, generator=g)
    with torch.no_grad():
        verts, jtr, _, _ = layer(pose, th_betas=betas, th_trans=trans)
    mods = RL.modules()
    faces = torch.from_numpy(smplh["faces"])
    normals = mods["data.tools"].vertex_normals(verts, faces.unsqueeze(0).repeat(Fn, 1, 1))
    y = (verts[:, ::23][:, :256] * 1.03).contiguous()
    p2p = mods["tools"].point2point_signed(verts, y, x_normals=normals, return_vector=True)
    sub = slice(None, None, 53)
    np.savez_compressed(os.path.join(OUT, "geometry.npz"), pose=pose.numpy(), betas=betas.numpy(), trans=trans.numpy(),
                        verts_sub=verts[:, sub].numpy(), jtr=jtr.numpy(), normals_sub=normals[:, sub].numpy(), y=y.numpy(),
                        y2x_signed=p2p[0].numpy(), yidx=p2p[2].numpy().astype(np.int32), y2x=p2p[4].numpy())

    # ---- the reference's own denoised_fn source (eval_smpl_short.py:84-130), random projector weights
    psd = projector_weights("random")
    proj, _ = RL.build_obj_projector(state_dict=psd, past_len=10, future_len=20)
    T, B = 30, 2
    b = S.make_smpl_batch(B=B, T=T)
    path = os.path.join(RL.ref_root(), "interdiff", "eval_smpl_short.py")
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "denoised_fn"][0]
    env = dict(torch=torch, args=Namespace(smpl_dim=132, past_len=10, future_len=20), rotation_6d_to_matrix=tf.rotation_6d_to_matrix,
               matrix_to_axis_angle=tf.matrix_to_axis_angle, markerset_ssm67_smplh=mods["data.utils"].markerset_ssm67_smplh,
               vertex_normals=mods["data.tools"].vertex_normals, point2point_signed=mods["tools"].point2point_signed)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), env)
    gt = torch.from_numpy(b["gt"])
    x = gt + 0.02 * torch.randn(gt.shape, generator=torch.Generator().manual_seed(4))
    kw = {"y": {"inpainted_motion": gt, "hand_pose": torch.from_numpy(b["hand_pose"]), "smpl": layer, "beta": torch.from_numpy(b["betas"]),
                "obj_model": Namespace(model=proj), "obj_points": torch.from_numpy(b["obj_points"])}}
    with torch.no_grad():
        o450 = env["denoised_fn"](x.clone(), torch.full((B,), 450), kw)
        o0 = env["denoised_fn"](x.clone(), torch.full((B,), 0), kw)
    # ---- evaluation metrics: the reference's own `metrics` function compiled out of eval_smpl_short.py
    from oracle import transforms as tfm
    from tests.helpers import metrics_inputs
    path = os.path.join(RL.ref_root(), "interdiff", "eval_smpl_short.py")
    fn = [n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == "metrics"][0]
    env = {"torch": torch, "axis_angle_to_matrix": tfm.axis_angle_to_matrix, "axis_angle_to_quaternion": tfm.axis_angle_to_quaternion,
           "vertex_normals": RL.modules()["data.tools"].vertex_normals, "point2point_signed": RL.modules()["tools"].point2point_signed}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), env)
    with torch.no_grad():
        mref = env["metrics"](**metrics_inputs(S.make_smplh_model(233)))
    np.savez_compressed(os.path.join(OUT, "metrics.npz"), **{k: v.numpy() for k, v in mref.items()})
    np.savez_compressed(os.path.join(OUT, "denoised_fn_random.npz"), x=x.numpy(), out450=o450.numpy(), out0=o0.numpy())
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


LBS_VERTEX_STRIDE = 16      # smplh_lbs.npz keeps every 16th vertex (and every joint) of the reference's SMPL layer output


def lbs_inputs():
    """seeded inputs of the SMPL-H layer comparison (tests/test_oracle_vs_reference.py::test_smplh_lbs)"""
    g = torch.Generator().manual_seed(1)
    Fn = 7
    pose = 0.4 * torch.randn(Fn, 156, generator=g)
    pose[0, 3:6] = 0  # exercise the |aa + 1e-8| small-angle path
    return pose, torch.randn(Fn, 10, generator=g), torch.randn(Fn, 3, generator=g)


def smooth_inputs():
    """seeded inputs of the `smooth` comparison (tests/test_oracle_vs_reference.py::test_smooth_and_best_of_samples)"""
    g = torch.Generator().manual_seed(0)
    return g, [torch.randn(30, 2, n, generator=g) for n in (6, 159, 12, 9, 3)]


def reference_lbs(smplh_np):
    pose, betas, trans = lbs_inputs()
    with torch.no_grad():
        v, j, _, _ = RL.build_smpl_layer(smplh_np)(pose, th_betas=betas, th_trans=trans)
    return v, j


def reference_smooth():
    path = os.path.join(RL.ref_root(), "interdiff", "eval_smpl_short.py")
    fn = [n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == "smooth"][0]
    env = {"args": Namespace(future_len=20)}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), env)
    return env["smooth"](*[x.clone() for x in smooth_inputs()[1]])


def main_host_side():
    """smplh_lbs.npz / smooth.npz: outputs of the reference's SMPL layer and of its `smooth`, for the tests that pin the
    oracle's LBS and the host-side post-processing where the reference tree is not installed"""
    v, j = reference_lbs(S.make_smplh_model(233))
    np.savez_compressed(os.path.join(OUT, "smplh_lbs.npz"), verts=v[:, ::LBS_VERTEX_STRIDE].numpy(), jtr=j.numpy())
    np.savez_compressed(os.path.join(OUT, "smooth.npz"), **{"out%d" % i: o.numpy() for i, o in enumerate(reference_smooth())})


if __name__ == "__main__":
    if "--host-side" in sys.argv:
        main_host_side()
    else:
        main()
        main_host_side()
