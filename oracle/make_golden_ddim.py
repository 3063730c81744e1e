"""Generate tests/golden/ddim_smpl_{random,ref}.npz from the reference's OWN DDIM sampler (imported via oracle.shims) --
run where the reference tree is installed:  python -m oracle.make_golden_ddim
TEST INFRASTRUCTURE, the DDIM counterpart of oracle/make_golden.py: seeded synthetic inputs (interdiff_b200.synthetic),
seeded random-init weights or the shipped checkpoint (oracle/_ref/weights).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from interdiff_b200 import synthetic as S  # noqa: E402
from oracle import ref_loader as RL  # noqa: E402
from tests.helpers import mdm_weights  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


DDIM_STEPS, DDIM_SPACING, DDIM_B, DDIM_T = 100, "ddim10", 4, 30
DDIM_CASES = [(eta, clip) for eta in (0.0, 0.5) for clip in (False, True)]


def ddim_key(eta, clip):
    return "eta%g_clip%d" % (eta, int(clip))


def reference_ddim_diffusion(steps=DDIM_STEPS, spacing=DDIM_SPACING):
    """the reference's own SpacedDiffusion, as create_gaussian_diffusion builds it (model/diffusion_smpl.py:250-284) but with
    the "ddimN" respacing its comment mentions (:256)"""
    gd, rs = RL.modules()["diffusion.gaussian_diffusion"], RL.modules()["diffusion.respace"]
    return rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(steps, spacing), betas=gd.get_named_beta_schedule("cosine", steps, 1.0),
                              model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_SMALL,
                              loss_type=gd.LossType.MSE, rescale_timesteps=False)


def reference_ddim_loop(diffusion, model, tape, kw, eta, clip):
    """SpacedDiffusion.ddim_sample_loop from x_T = tape[0]; the per-step th.randn_like (:779) returns tape[k + 1]"""
    gd = RL.modules()["diffusion.gaussian_diffusion"]
    idx = [0]

    def fake(x):
        idx[0] += 1
        return tape[idx[0]].clone()
    old, gd.th.randn_like = gd.th.randn_like, fake
    try:
        with torch.no_grad():
            return diffusion.ddim_sample_loop(model, tuple(tape[0].shape), noise=tape[0].clone(), clip_denoised=clip, model_kwargs=kw, eta=eta)
    finally:
        gd.th.randn_like = old


def main_ddim():
    """ddim_smpl_{random,ref}.npz: the reference's DDIM loop (ddim_sample, gaussian_diffusion.py:738-999) on a 100-step cosine
    schedule respaced "ddim10", B=4, T=30, inpainted past, seeded tape, for eta in {0, 0.5} x clip_denoised in {False, True}.
    With the shipped checkpoint (ddim_smpl_ref.npz) each case is stored twice: the reference as it runs (float32, key eta<e>_clip<c>) and the same classes in float64
    (model.double(), float64 inputs; key + "_f64", stored as float32).  With the shipped checkpoint the two differ by up to a few 1e-2: the
    chain amplifies the reference's own rounding, and that distance is what parity against the float32 run is judged by."""
    diffusion = reference_ddim_diffusion()
    for source in ("random", "ref"):
        sd = mdm_weights("smpl", source)
        model, _, _ = RL.build_mdm_smpl(state_dict=sd, diffusion_steps=DDIM_STEPS)
        b = S.make_smpl_batch(B=DDIM_B, T=DDIM_T)
        tape = torch.from_numpy(S.noise_tape(b["gt"].shape, diffusion.num_timesteps))
        kw = {"y": {"cond": torch.from_numpy(b["cond"]), "inpainted_motion": torch.from_numpy(b["gt"]),
                    "inpainting_mask": torch.from_numpy(b["mask"])}}
        out = {ddim_key(eta, clip): reference_ddim_loop(diffusion, model, tape, kw, eta, clip).numpy() for eta, clip in DDIM_CASES}
        if source == "random":      # seeded weights: a well-conditioned chain (float32 and float64 agree to ~2e-6)
            np.savez_compressed(os.path.join(OUT, "ddim_smpl_%s.npz" % source), timestep_map=np.asarray(diffusion.timestep_map), **out)
            continue
        model.double()
        kw64 = {"y": {"cond": kw["y"]["cond"].double(), "inpainted_motion": kw["y"]["inpainted_motion"].double(),
                      "inpainting_mask": kw["y"]["inpainting_mask"]}}
        for eta, clip in DDIM_CASES:
            # stored rounded to float32 (6e-8 relative: far below the distances it is used for)
            out[ddim_key(eta, clip) + "_f64"] = reference_ddim_loop(diffusion, model, tape.double(), kw64, eta, clip).float().numpy()
        np.savez_compressed(os.path.join(OUT, "ddim_smpl_%s.npz" % source), timestep_map=np.asarray(diffusion.timestep_map), **out)
        print("ddim_smpl_%s.npz" % source, os.path.getsize(os.path.join(OUT, "ddim_smpl_%s.npz" % source)))


if __name__ == "__main__":
    main_ddim()
