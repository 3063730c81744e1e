"""Round-2 probe (runs on the GPU box): sampling-loop graph modes, config 3, and the SMPL-H LBS paths
(tensor-core pose blend + sparse / dense skinning vs the fp32 SIMT kernel) with CUDA events."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200 import synthetic as S  # noqa: E402
from interdiff_b200.diffusion.gaussian_diffusion import get_named_beta_schedule  # noqa: E402
from interdiff_b200.engine import Engine  # noqa: E402
from interdiff_b200.weights import bench_weights  # noqa: E402

B, T, steps = 64, 30, 100
eng = Engine("cuda:0")
eng.load_denoiser(bench_weights("diffusion_smpl"), "smpl")
b = S.make_smpl_batch(B=B, T=T)
eng.bind(b["cond"], T)
eng.init_diffusion(get_named_beta_schedule("cosine", steps))
tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps)).cuda()
gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")


def timed(fn, n=5, warm=2, flush_l2=False):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(n):
        if flush_l2:
            flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / n


for mode in ("off", "step", "loop"):
    ms = timed(lambda: eng.p_sample_loop(tape, gt, mask, use_graph=mode), n=8, warm=3, flush_l2=True)
    print("config 2, graph mode %-4s: %.3f ms / 100 steps -> %.0f steps/s (%.1f us/step)" % (mode, ms, 100e3 / ms, ms * 10))

F = T * B
g = torch.Generator().manual_seed(0)
pose = (0.3 * torch.randn(F, 156, generator=g)).cuda()
betas = torch.randn(F, 10, generator=g).cuda()
trans = torch.randn(F, 3, generator=g).cuda()
byt = 41.7e6 + F * 84.0e3
for wname, sparse in (("dense tail (every bone non-zero)", False), ("<= 4 non-zero bones per vertex (as SMPL-H)", True)):
    eng.load_body(S.make_smplh_model(233, sparse_weights=sparse))
    for backend in ("simt", "tcgen05"):
        eng.set_gemm_backend(backend)
        ms = timed(lambda: eng.lbs(pose, betas, trans, want_jtr=False), n=10, warm=3, flush_l2=True)
        print("LBS F=%d, weights: %s, %s path: %.3f ms ; algorithmic %.1f MB -> %.0f GB/s (%.1f %% of the 3350 GB/s data-sheet HBM3 rate) ; %.1f GFLOP -> %.1f TFLOP/s" % (
            F, wname, "fp32 SIMT" if backend == "simt" else "wgmma blend + skinning", ms, byt / 1e6, byt / ms / 1e6, byt / ms / 1e6 / 33.50,
            F * 33.2e-3, F * 33.2e6 / ms / 1e9))
eng.set_gemm_backend("tcgen05")
eng.load_body(S.make_smplh_model(233, sparse_weights=True))
for mc in (False, True):
    eng.set_gemm_multicast(mc)
    ms = timed(lambda: eng.lbs(pose, betas, trans, want_jtr=False), n=10, warm=3, flush_l2=True)
    print("LBS F=%d sparse weights, blend GEMM %s multicast row-tile pairs: %.3f ms (%.0f GB/s)" % (F, "with" if mc else "without", ms, byt / ms / 1e6))
eng.set_gemm_multicast(True)

if "--config3" in sys.argv:
    from interdiff_b200.weights import bench_weights as bw
    eng.load_body(S.make_smplh_model(233, sparse_weights=True))
    eng.load_projector(bw("correction_smpl"), 10, 20)
    eng.bind_correction(b["hand_pose"], b["betas"], b["obj_points"], past_len=10)
    for mode in ("step", "loop"):
        ms2 = timed(lambda: eng.p_sample_loop(tape, gt, mask, correction=False, use_graph=mode), flush_l2=True)
        ms3 = timed(lambda: eng.p_sample_loop(tape, gt, mask, correction=True, use_graph=mode), flush_l2=True)
        print("graph mode %s: config 2 %.2f ms, config 3 %.2f ms / 100 steps -> %.0f steps/s ; one correction step = %.2f ms" % (
            mode, ms2, ms3, 100e3 / ms3, (ms3 - ms2) / 2))
    verts, _ = eng.lbs(pose, betas, trans, want_jtr=False)
    ms = timed(lambda: eng.vertex_normals(verts))
    print("vertex_normals F=%d: %.3f ms" % (F, ms))
    normals = eng.vertex_normals(verts)
    obj = (verts[:, ::4][:, :2048] * 1.1).contiguous()
    ms = timed(lambda: eng.signed_nn(obj, verts, normals), n=3, warm=1)
    print("signed_nn (pruned) F=%d 2048x6890: %.3f ms" % (F, ms))
