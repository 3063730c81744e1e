"""Fused feed-forward cluster kernel vs float64 and vs the two-GEMM path: error and loop time.
usage: python profiles/mlp_probe.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200 import synthetic as S  # noqa: E402
from interdiff_b200.engine import Engine  # noqa: E402
from interdiff_b200.diffusion.gaussian_diffusion import get_named_beta_schedule  # noqa: E402
from tests.helpers import mdm_weights  # noqa: E402

eng = Engine("cuda:0")
g = torch.Generator().manual_seed(1)
for M in (1920, 100, 129):
    x = torch.randn(M, 256, generator=g)
    w1 = torch.randn(1024, 256, generator=g) / 16
    b1 = torch.randn(1024, generator=g) * 0.1
    w2 = torch.randn(256, 1024, generator=g) / 32
    b2 = torch.randn(256, generator=g) * 0.1
    res = torch.randn(M, 256, generator=g)
    ref = torch.nn.functional.gelu(x.double() @ w1.double().T + b1.double()) @ w2.double().T + b2.double() + res.double()
    outs = [eng.mlp(x, w1, b1, w2, b2, res).cpu() for _ in range(2)]
    print("M=%d: max-norm rel err vs fp64 %.3e, deterministic %s" % (M, ((outs[0].double() - ref).abs().max() / ref.abs().max()).item(),
                                                                    torch.equal(outs[0], outs[1])))
eng.load_denoiser(mdm_weights("smpl", "auto"), "smpl")
b = S.make_smpl_batch(B=64, T=30)
eng.bind(b["cond"], 30)
eng.init_diffusion(get_named_beta_schedule("cosine", 100))
tape = torch.from_numpy(S.noise_tape(b["gt"].shape, 100)).cuda()
gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
outs = {}
for on in (0, 2, 0, 2):
    eng.set_fused_mlp(on)
    for _ in range(2):
        out = eng.p_sample_loop(tape, gt, mask)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        out = eng.p_sample_loop(tape, gt, mask)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    outs[on] = out.clone()
    print("fused mlp %d: %.3f ms / 100 steps -> %.1f steps/s" % (on, ms, 100e3 / ms))
print("max-norm rel diff of the 100-step samples between two GEMMs and the fused kernel: %.3e" % (
    ((outs[0] - outs[2]).abs().max() / outs[0].abs().max()).item()))
