"""Conditioning probe of the free-running sampling loop (TEST INFRASTRUCTURE; runs where /root/reference exists).

BASELINE configs[1] exactly (SMPL diffusion, B=64, T=30, 100-step cosine schedule, shipped diffusion.ckpt, inpainted
past, identical noise tape) through the REFERENCE's own classes (MDM + SpacedDiffusion.p_sample via oracle/shims.py):

  curve "self"   : reference with 1 thread  vs  reference with N threads      (same code, different reduction order)
  curve "f64"    : reference in float32     vs  the SAME reference classes in float64 (model.double(), double inputs):
                   the rounding error of the reference itself, amplified by the chain - the yardstick that does not
                   involve any code of this repository
  curve "oracle" : oracle.restate (N threads) vs reference (N threads); "oracle_f64": oracle.restate vs reference float64

per step k = 0..99 (timestep i = 99 - k): max|a-b| / max|b| of the sample x_{t-1} after that step.  The output
(tests/golden/conditioning_probe.json + .txt) is what tests/test_gpu_configs.py::test_config2_full_loop reads to decide up
to which step a free-running comparison at 1e-3 is meaningful: the first step where the reference disagrees with
ITSELF (float32 vs float64, or 1 vs N threads, whichever comes first) by more than 1e-4 (SURVEY 8d "Parity check",
VERDICT r1 "What's weak" 1).

  python -m oracle.conditioning_probe [--B 64] [--threads 8] [--out tests/golden/conditioning_probe]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-12)).item()


def reference_trajectory(model, diffusion, tape, gt, mask, cond, threads, dtype=torch.float32):
    torch.set_num_threads(threads)
    n = diffusion.num_timesteps
    tape, gt, cond = tape.to(dtype), gt.to(dtype), cond.to(dtype)
    x = tape[0].clone()
    kw = {"y": {"cond": cond, "inpainted_motion": gt, "inpainting_mask": mask}}
    out = []
    # p_sample draws th.randn_like(x) itself (gaussian_diffusion.py:532): feed the tape through the RNG hook below
    orig = torch.randn_like
    for k, i in enumerate(reversed(range(n))):
        t = torch.full((x.shape[0],), i, dtype=torch.long)
        torch.randn_like = lambda _x, _k=k: tape[_k + 1]
        try:
            with torch.no_grad():
                x = diffusion.p_sample(model, x, t, clip_denoised=False, model_kwargs=kw)["sample"]
        finally:
            torch.randn_like = orig
        out.append(x.clone())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "conditioning_probe"))
    a = ap.parse_args()
    from interdiff_b200 import synthetic as S
    from oracle import ref_loader as RL
    from oracle import restate as R
    model, diffusion, _ = RL.build_mdm_smpl(diffusion_steps=a.steps)
    _, sd = RL.load_ckpt("diffusion")
    b = S.make_smpl_batch(B=a.B, T=a.T)
    gt, mask, cond = torch.from_numpy(b["gt"]), torch.from_numpy(b["mask"]), torch.from_numpy(b["cond"])
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, a.steps))
    t0 = time.time()
    ref_n = reference_trajectory(model, diffusion, tape, gt, mask, cond, a.threads)
    t1 = time.time()
    ref_1 = reference_trajectory(model, diffusion, tape, gt, mask, cond, 1)
    t2 = time.time()
    ref_64 = reference_trajectory(model.double(), diffusion, tape, gt, mask, cond, a.threads, torch.float64)
    model.float()
    t2b = time.time()
    torch.set_num_threads(a.threads)
    tables = R.diffusion_tables(R.named_beta_schedule("cosine", a.steps))
    with torch.no_grad():
        _, traj = R.p_sample_loop(lambda x, t: R.mdm_smpl_forward(sd, x, t, cond, faithful=False), tables, tape, gt, mask,
                                  return_trajectory=True)
    t3 = time.time()
    self_curve = [rel(x1, xn) for x1, xn in zip(ref_1, ref_n)]
    f64_curve = [rel(xn, x64) for xn, x64 in zip(ref_n, ref_64)]
    oracle_curve = [rel(o[0], xn) for o, xn in zip(traj, ref_n)]
    oracle64_curve = [rel(o[0], x64) for o, x64 in zip(traj, ref_64)]
    first = next((k for k, (v, w) in enumerate(zip(self_curve, f64_curve)) if max(v, w) > 1e-4), len(self_curve))
    res = dict(config="BASELINE configs[1]: SMPL diffusion, B=%d, T=%d, %d-step cosine schedule, diffusion.ckpt, noise tape seed 233" % (a.B, a.T, a.steps),
               threads=a.threads, seconds=dict(reference_N=t1 - t0, reference_1=t2 - t1, reference_f64=t2b - t2, oracle_N=t3 - t2b),
               self_disagreement=self_curve, reference_f32_vs_f64=f64_curve, oracle_vs_reference=oracle_curve,
               oracle_vs_reference_f64=oracle64_curve, first_step_self_above_1e4=first,
               metric="max|a-b|/max|b| of the sample after step k (timestep i = steps-1-k)")
    with open(a.out + ".json", "w") as f:
        json.dump(res, f, indent=1)
    with open(a.out + ".txt", "w") as f:
        f.write("# %s\n# self = reference 1 thread vs %d threads | f64 = reference float32 vs float64 | oracle = oracle.restate vs reference | "
                "oracle64 = oracle.restate vs reference float64\n" % (res["config"], a.threads))
        f.write("# first step where the reference disagrees with itself (threads or precision) by > 1e-4: k = %d (timestep %d)\n" % (first, a.steps - 1 - first))
        f.write("# step k  timestep   self        f64         oracle      oracle64\n")
        for k in range(len(self_curve)):
            f.write("%7d  %8d   %.3e   %.3e   %.3e   %.3e\n" % (k, a.steps - 1 - k, self_curve[k], f64_curve[k], oracle_curve[k], oracle64_curve[k]))
    print(json.dumps({k: v for k, v in res.items() if not isinstance(v, list)}))


if __name__ == "__main__":
    main()
