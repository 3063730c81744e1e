"""The skeleton evaluation path of eval_skeleton.py (sample_once_proj, :114-142) on one GPU: prints one JSON line.

Shapes of the shipped skeleton configuration: B=64, T=20 (past_len 10, future_len 10), 1000-step cosine schedule, the
shipped checkpoints where they are exported under oracle/_ref/weights, seeded weights otherwise.
  * `_get_embeddings` (the conditioning encoder, idb_encode_condition_skeleton, + the gt concatenation): mean ms per call
    over --calls calls, CUDA events around the calls, after warm-up;
  * one sample_once_proj call with the correction hook as the script's plain Python callback (step by step) and as
    sampling.FusedSkeletonCorrection (the whole loop in the library): ms per call, host clock around work that ends in a
    device synchronise, after one warm-up call of each.
The device line (name, power limit, max SM clock) is read with a read-only nvidia-smi query.

  python profiles/skeleton_eval_probe.py [--calls 50] [--loops 2]
"""
import argparse
import json
import os
import sys
import time
from argparse import Namespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from interdiff_b200 import synthetic as S  # noqa: E402
from interdiff_b200 import weights as W  # noqa: E402
from interdiff_b200.model.correction_skeleton import ObjProjector  # noqa: E402
from interdiff_b200.model.diffusion_skeleton import create_model_and_diffusion  # noqa: E402
from interdiff_b200.sampling import FusedSkeletonCorrection  # noqa: E402
from profiles.sampler_bench import device_line  # noqa: E402

ARGS = dict(embedding_dim=256, smpl_dim=63, num_joints=21, num_points=12, dropout=0.0, num_heads=4, ff_size=256, activation="gelu",
            latent_usage="memory", past_len=10, future_len=10, cond_mask_prob=0, diffusion_steps=1000, noise_schedule="cosine",
            sigma_small=True, weight_v=1)


def _load(module, sd):
    own = module.state_dict()
    module.load_state_dict({k: (sd[k].reshape(own[k].shape) if k in sd else v) for k, v in own.items()})
    return module.cuda().eval()


def quat_to_matrix(q):
    """pytorch3d quaternion_to_matrix (real part first)"""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def script_denoised_fn(x, t, model_kwargs):
    """eval_skeleton.py:80-111 (its unused body_obj_to_contact left out)"""
    if t[0] > 500 or t[0] % 50 != 0:
        return x
    body_pred, _, _ = torch.split(x.squeeze(1).permute(2, 0, 1).contiguous(), [63, 36, 7], dim=2)
    _, _, pose_gt = torch.split(model_kwargs["y"]["inpainted_motion"].squeeze(1).permute(2, 0, 1).contiguous(), [63, 36, 7], dim=2)
    T, B, _ = body_pred.shape
    trans_gt, angles_gt = torch.split(pose_gt, [3, 4], dim=2)
    angles, trans = model_kwargs["y"]["obj_model"].model.sample(angles_gt, trans_gt, body_pred.view(T, B, -1, 3))
    pose = torch.cat([trans, angles], dim=2)
    rot = quat_to_matrix(torch.cat([pose[:, :, -1, None], pose[:, :, -4:-1]], dim=2))[:, :, None]
    obj = (rot.matmul(model_kwargs["zero_pose_obj"][None, :, :, :, None]) + pose[:, :, None, :3, None])[..., 0].reshape(T, B, -1)
    x_ = torch.cat([body_pred, obj, pose], dim=2).permute(1, 2, 0).unsqueeze(1).contiguous()
    return t[0] / 1000 * x + (1 - t[0] / 1000) * x_


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--loops", type=int, default=2)
    a = ap.parse_args()
    B, T, P = 64, 20, 10
    model, diffusion = create_model_and_diffusion(Namespace(**ARGS))
    shipped = W.have_ref_weights("diffusion_skeleton_encoder") and W.have_ref_weights("diffusion_skeleton")
    model = _load(model, {**W.bench_weights("diffusion_skeleton"), **W.bench_weights("diffusion_skeleton_encoder")})
    proj = _load(ObjProjector(Namespace(num_joints=21, dropout=0.0, past_len=P, future_len=T - P, embedding_dim=128)),
                 W.bench_weights("correction_skeleton"))
    b = S.make_skeleton_batch(B=B, T=T, past_len=P)
    xs = torch.from_numpy(b["gt"]).squeeze(1).permute(2, 0, 1)
    batch = [xs[..., :63].reshape(T, B, 21, 3).transpose(0, 1).contiguous(), xs[..., 63:99].reshape(T, B, 12, 3).transpose(0, 1).contiguous(),
             xs[..., 99:].transpose(0, 1).contiguous(), torch.from_numpy(b["zero_pose_obj"])]
    dev = torch.device("cuda:0")
    body_gt, obj_gt, pose_gt = (x.transpose(0, 1).float().to(dev) for x in batch[:3])
    zp = batch[3].float().to(dev)
    with torch.no_grad():
        for _ in range(3):
            embedding, gt = model._get_embeddings(body_gt, obj_gt, pose_gt, zp)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.calls):
            embedding, gt = model._get_embeddings(body_gt, obj_gt, pose_gt, zp)
        e1.record()
        torch.cuda.synchronize()
        emb_ms = e0.elapsed_time(e1) / a.calls
        gt = gt.permute(1, 2, 0).unsqueeze(1).contiguous()
        mask = torch.ones_like(gt, dtype=torch.bool)
        mask[:, :, :, P:] = False
        kw = {"y": {"cond": embedding, "inpainted_motion": gt, "inpainting_mask": mask, "obj_model": Namespace(model=proj)},
              "zero_pose_obj": zp}
        res = {}
        for name, fn in (("python_callback", script_denoised_fn), ("fused", FusedSkeletonCorrection())):
            times = []
            for k in range(a.loops + 1):
                noise = torch.randn(*gt.shape, device=dev)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                diffusion.p_sample_loop(model, gt.shape, clip_denoised=False, noise=noise, model_kwargs=kw, denoised_fn=fn)
                torch.cuda.synchronize()
                if k:
                    times.append((time.perf_counter() - t0) * 1e3)
            res[name] = dict(ms_per_call=min(times), all_ms=times)
    print(json.dumps(dict(probe="skeleton_eval", device=device_line(), B=B, T=T, steps=1000, weights="shipped" if shipped else "seeded",
                          get_embeddings_ms=emb_ms, sample_once_proj=res,
                          speedup_fused_vs_callback=res["python_callback"]["ms_per_call"] / res["fused"]["ms_per_call"])))


if __name__ == "__main__":
    main()
