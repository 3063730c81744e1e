"""Conditioning probe of the deterministic DDIM chain (TEST INFRASTRUCTURE; a CPU run where the reference tree is installed), the DDIM
counterpart of oracle/conditioning_probe.py.

BASELINE configs[1] shapes (SMPL diffusion, B=64, T=30, inpainted past, shipped diffusion.ckpt) on the 100-step cosine
schedule respaced "ddim50" and "ddim10", through the reference's own SpacedDiffusion.ddim_sample at eta = 0 (deterministic:
x_T = noise tape entry 0, no other noise), reference float32 vs the same classes in float64.  Per spacing: the curve
max|a-b|/max|b| of the sample after each step and the first step where it exceeds 1e-4.  Written to
tests/golden/ddim_conditioning.json (read by tests/test_gpu_ddim.py::test_ddim50_free_running_configs1 to decide up to
which step a free-running comparison at 1e-3 is meaningful).

  python -m oracle.ddim_conditioning_probe [--B 64] [--threads 8] [--out tests/golden/ddim_conditioning]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.conditioning_probe import rel  # noqa: E402


def reference_ddim_trajectory(model, diffusion, x_T, gt, mask, cond, threads, dtype=torch.float32):
    """SpacedDiffusion.ddim_sample (gaussian_diffusion.py:738-788) at eta = 0, step by step from x_T"""
    torch.set_num_threads(threads)
    x, gt, cond = x_T.to(dtype), gt.to(dtype), cond.to(dtype)
    kw = {"y": {"cond": cond, "inpainted_motion": gt, "inpainting_mask": mask}}
    out = []
    for i in reversed(range(diffusion.num_timesteps)):
        with torch.no_grad():
            x = diffusion.ddim_sample(model, x, torch.full((x.shape[0],), i, dtype=torch.long), clip_denoised=False, model_kwargs=kw,
                                      eta=0.0)["sample"]
        out.append(x.clone())
    return out


def main_ddim(a):
    from interdiff_b200 import synthetic as S
    from oracle import make_golden_ddim as MG
    from oracle import ref_loader as RL
    model, _, _ = RL.build_mdm_smpl(diffusion_steps=a.steps)
    b = S.make_smpl_batch(B=a.B, T=a.T)
    gt, mask, cond = torch.from_numpy(b["gt"]), torch.from_numpy(b["mask"]), torch.from_numpy(b["cond"])
    x_T = torch.from_numpy(S.noise_tape(b["gt"].shape, a.steps))[0]
    res = dict(config="BASELINE configs[1] shapes: SMPL diffusion, B=%d, T=%d, %d-step cosine schedule respaced, diffusion.ckpt, "
                      "DDIM eta = 0, x_T = noise tape seed 233 entry 0" % (a.B, a.T, a.steps),
               threads=a.threads, metric="max|a-b|/max|b| of the sample after step k (step index i = n-1-k), reference float32 vs float64",
               spacings={})
    for spacing in ("ddim50", "ddim10"):
        diffusion = MG.reference_ddim_diffusion(a.steps, spacing)
        t0 = time.time()
        r32 = reference_ddim_trajectory(model.float(), diffusion, x_T, gt, mask, cond, a.threads)
        t1 = time.time()
        r64 = reference_ddim_trajectory(model.double(), diffusion, x_T, gt, mask, cond, a.threads, torch.float64)
        t2 = time.time()
        model.float()
        curve = [rel(x, y) for x, y in zip(r32, r64)]
        first = next((k for k, v in enumerate(curve) if v > 1e-4), len(curve))
        res["spacings"][spacing] = dict(n=diffusion.num_timesteps, timestep_map=list(diffusion.timestep_map), reference_f32_vs_f64=curve,
                                        first_step_above_1e4=first, seconds=dict(reference_f32=t1 - t0, reference_f64=t2 - t1))
        print(spacing, "first step above 1e-4:", first, "final:", curve[-1])
    with open(a.out + ".json", "w") as f:
        json.dump(res, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "ddim_conditioning"))
    main_ddim(ap.parse_args())


if __name__ == "__main__":
    main()
