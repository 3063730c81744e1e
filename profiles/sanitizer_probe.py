"""Small end-to-end exercise of every kernel family for compute-sanitizer (memcheck / racecheck):
3-step sampling loop (graph off), fused feed-forward, GEMM tile configurations, LBS, normals, pruned NN, correction."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200 import synthetic as S  # noqa: E402
from interdiff_b200.diffusion.gaussian_diffusion import get_named_beta_schedule  # noqa: E402
from interdiff_b200.engine import Engine  # noqa: E402
from tests.helpers import encoder_weights, metrics_inputs, projector_weights  # noqa: E402

B, T, steps = 3, 30, 3
eng = Engine("cuda:0")
if os.environ.get("IDB_SPLIT_ATTN"):      # standard layers' self- / cross-attention as two launches (racecheck cannot see that the fused
    eng.set_fused_mlp(10)                 # kernel's two staging phases on the same shared memory are ordered by mbarrier waits)
eng.load_denoiser(encoder_weights("random"), "smpl")
smplh = S.make_smplh_model(233)
eng.load_body(smplh)
eng.load_projector(projector_weights("random"), 10, 20)
b = S.make_smpl_batch(B=B, T=T)
eng.bind(b["cond"], T)
eng.bind_correction(b["hand_pose"], b["betas"], b["obj_points"], past_len=10)
eng.init_diffusion(get_named_beta_schedule("cosine", steps))
tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps)).cuda()
gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
out = eng.p_sample_loop(tape, gt, mask, correction=True, use_graph=False)
out2 = eng.p_sample_loop(tape, gt, mask, correction=False, use_graph=True)
g = torch.Generator().manual_seed(0)
for (M, N, K) in ((200, 1536, 256), (130, 256, 1024), (70, 72, 36)):
    eng.gemm(torch.randn(M, K, generator=g), torch.randn(N, K, generator=g), bias=torch.randn(N, generator=g), gelu=True)
eng.gemm(torch.randn(130, 1024, generator=g), torch.randn(256, 1024, generator=g), split_k=True)
eng.mlp(torch.randn(129, 256, generator=g), torch.randn(1024, 256, generator=g) / 16, torch.randn(1024, generator=g),
        torch.randn(256, 1024, generator=g) / 32, torch.randn(256, generator=g), torch.randn(129, 256, generator=g))
# conditioning path (PointNet++ + encoder), metrics, both fused feed-forward levels
pts = 0.2 * (torch.rand(B, 2048, 3, generator=g) - 0.5)
pc = eng.pointcloud_embed(pts.cuda())
cond = eng.encode_condition(gt[..., :10].contiguous(), pc)
for level in (2, 0):
    eng.set_fused_mlp(level)
    eng.bind(cond, T)
    eng.forward(tape[0], torch.tensor([5, 500, 999]).cuda())
eng.set_fused_mlp(2)
mi = metrics_inputs(smplh, T=3, B=2, P=128)
eng.metrics(**{k: v.cuda() for k, v in mi.items() if k != "faces"})
lw, lb = torch.ones(256), torch.zeros(256)
eng.mlp(torch.randn(129, 256, generator=g), torch.randn(1024, 256, generator=g) / 16, torch.randn(1024, generator=g),
        torch.randn(256, 1024, generator=g) / 32, torch.randn(256, generator=g), torch.randn(129, 256, generator=g), ln_w=lw, ln_b=lb)
# round 2: whole-loop graph, tensor-core LBS (sparse and dense skinning, multicast and plain blend GEMM, partial row tiles),
# rollout step, post-processing, skeleton correction net + hook
out3 = eng.p_sample_loop(tape, gt, mask, correction=True, use_graph="loop")
for sparse in (True, False):
    eng.load_body(S.make_smplh_model(233, sparse_weights=sparse))
    for mc in (True, False):
        eng.set_gemm_multicast(mc)
        eng.lbs(0.3 * torch.randn(300, 156, generator=g), torch.randn(300, 10, generator=g), torch.randn(300, 3, generator=g))
eng.set_gemm_multicast(True)
body = torch.randn(T, B, 159, generator=g); obj = torch.randn(T, B, 6, generator=g); jtr = torch.randn(T, B, 52, 3, generator=g)
ngt, cen = eng.rollout_next_window(body, obj, jtr, T, 10)
eng.add_offset_(jtr.cuda().contiguous(), cen)
x = torch.randn(T, B, 7, 3, generator=g).cuda()
eng.smooth_(x, 20)
eng.metric_min_(torch.full((6, B), 1e10, device="cuda"), torch.rand(6, B, generator=g))
from tests.helpers import mdm_weights, projector_skeleton_weights  # noqa: E402
eng.load_projector_skeleton(projector_skeleton_weights("random"), 10, 10, n_joints=21)
eng.projector_sample_skeleton(torch.randn(20, B, 4, generator=g), torch.randn(20, B, 3, generator=g), torch.randn(20, B, 21, 3, generator=g))
bs = S.make_skeleton_batch(B=2, T=20)
eng.load_denoiser(mdm_weights("skeleton", "random"), "skeleton")
eng.bind(bs["cond"], 20, zero_pose_obj=bs["zero_pose_obj"])
eng.init_diffusion(get_named_beta_schedule("cosine", 2))
tp = torch.from_numpy(S.noise_tape(bs["gt"].shape, 2)).cuda()
out4 = eng.p_sample_loop(tp, torch.from_numpy(bs["gt"]).cuda(), torch.from_numpy(bs["mask"]).cuda(), correction=True, use_graph="off")
torch.cuda.synchronize()
print("sanitizer probe done", float(out.abs().max()), float(out2.abs().max()), float(out3.abs().max()), float(out4.abs().max()))
