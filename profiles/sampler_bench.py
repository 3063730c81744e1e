"""DDPM vs DDIM sampling throughput on one GPU: prints one JSON line.

configs[1] shapes (SMPL diffusion, B=64, T=30, inpainted past, 100-step cosine schedule; the shipped checkpoint where it is
exported under oracle/_ref/weights, seeded weights otherwise):
  * DDPM-100 through idb_p_sample_loop (noise tape), and DDIM "ddim50" / "ddim25" / "ddim10" at eta = 0 through
    idb_ddim_sample_loop without a tape, each as the whole loop in one CUDA graph;
  * per sampler: ms per sampling call (CUDA events around each call, warm-up first, a 256 MB fill evicts L2 between timed
    calls outside the event pair, as bench.py does), denoising steps/s and samples/s.
At the configs[3] shape (B=256, T=30, 1000-step schedule) it also reports torch.cuda.max_memory_allocated for a DDPM-1000
loop with its noise tape and for the tape-free DDIM loop of the same schedule (eta = 0, no respacing).
The device line (name, power limit, max SM clock) is read with a read-only nvidia-smi query.

  python profiles/sampler_bench.py [--calls 10] [--warmup 3] [--skip-memory]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from interdiff_b200 import synthetic as S  # noqa: E402
from interdiff_b200.diffusion.gaussian_diffusion import get_named_beta_schedule  # noqa: E402
from interdiff_b200.diffusion.respace import SpacedDiffusion, space_timesteps  # noqa: E402
from interdiff_b200.engine import Engine  # noqa: E402
from interdiff_b200.sampling import draw_tape  # noqa: E402
from interdiff_b200.weights import bench_weights, load_ref_weights  # noqa: E402


def device_line(idx=0):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %r" % (e,)
    return {"query": q, "value": out, "torch_name": torch.cuda.get_device_name(idx)}


def spaced(n, spacing):
    """(betas, timestep_map) of SpacedDiffusion(space_timesteps(n, spacing)) over the cosine schedule"""
    from interdiff_b200.diffusion import gaussian_diffusion as gd
    d = SpacedDiffusion(space_timesteps(n, spacing), betas=get_named_beta_schedule("cosine", n), model_mean_type=gd.ModelMeanType.START_X,
                        model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    return d.betas, d.timestep_map


def time_calls(fn, calls, warmup, flush):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
    for s, e in ev:
        flush.fill_(1.0)
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    ms = sorted(s.elapsed_time(e) for s, e in ev)
    return dict(ms_mean=sum(ms) / len(ms), ms_median=ms[len(ms) // 2], ms_min=ms[0], ms_max=ms[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-memory", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench needs a CUDA device (sm_90a); nothing is measured on the CPU")
    dev = torch.device("cuda:0")
    eng = Engine(dev)
    eng.load_denoiser(bench_weights("diffusion_smpl"), "smpl")
    weights = "shipped checkpoint" if load_ref_weights("diffusion_smpl") is not None else "seeded random init"
    B, T, n = 64, 30, 100
    b = S.make_smpl_batch(B=B, T=T)
    gt, mask = torch.from_numpy(b["gt"]).to(dev), torch.from_numpy(b["mask"]).to(dev)
    eng.bind(torch.from_numpy(b["cond"]).to(dev), T)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    out = torch.empty(gt.shape, device=dev)
    torch.manual_seed(233)
    x_T = torch.randn(gt.shape, device=dev)
    res = dict(config="configs[1] shapes: SMPL diffusion, B=%d, T=%d, inpainted past, cosine schedule of %d steps" % (B, T, n),
               weights=weights, timing="CUDA events per call, %d warm-up calls, %d timed calls, L2 flushed before each" % (a.warmup, a.calls),
               graph="whole loop as one CUDA graph", samplers={})

    # ---- DDPM-100 (tape) vs DDIM-k (eta = 0, no tape); one engine, each sampler warmed up (and its graph captured) before timing
    eng.init_diffusion(get_named_beta_schedule("cosine", n))
    tape = draw_tape(eng, x_T, n, seed=233)
    t = time_calls(lambda: eng.p_sample_loop(tape, gt, mask, use_graph=True, out=out), a.calls, a.warmup, flush)
    res["samplers"]["ddpm100"] = dict(steps=n, entry="idb_p_sample_loop", **t)
    for k in (50, 25, 10):
        betas, tmap = spaced(n, "ddim%d" % k)
        eng.init_diffusion_ddim(betas, tmap, eta=0.0)
        t = time_calls(lambda: eng.ddim_sample_loop(x_T, None, gt, mask, use_graph=True, out=out), a.calls, a.warmup, flush)
        res["samplers"]["ddim%d" % k] = dict(steps=len(betas), entry="idb_ddim_sample_loop, eta 0, no tape", **t)
    for v in res["samplers"].values():
        v["steps_per_s"] = v["steps"] / (v["ms_mean"] / 1e3)
        v["samples_per_s"] = B / (v["ms_mean"] / 1e3)
    base = res["samplers"]["ddpm100"]["ms_mean"]
    for v in res["samplers"].values():
        v["speedup_vs_ddpm100"] = base / v["ms_mean"]
    del tape

    # ---- memory at configs[3] shape: B=256, 1000 steps; tape (1001 x B x 144 x 30 floats) vs none
    if not a.skip_memory:
        B3, n3 = 256, 1000
        del flush
        b3 = S.make_smpl_batch(B=B3, T=T)
        gt3, mask3 = torch.from_numpy(b3["gt"]).to(dev), torch.from_numpy(b3["mask"]).to(dev)
        eng.bind(torch.from_numpy(b3["cond"]).to(dev), T)
        x3 = torch.randn(gt3.shape, device=dev)
        out3 = torch.empty_like(x3)
        mem = {}
        for name in ("ddim1000_eta0_no_tape", "ddpm1000_tape"):
            eng._keep_loop = None          # the engine keeps the last loop's tensors alive until the next call
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            base_alloc = torch.cuda.memory_allocated(dev)
            if name.startswith("ddpm"):
                eng.init_diffusion(get_named_beta_schedule("cosine", n3))
                t3 = draw_tape(eng, x3, n3, seed=233)
                eng.p_sample_loop(t3, gt3, mask3, use_graph=True, out=out3)
                torch.cuda.synchronize()
                del t3
            else:
                eng.init_diffusion_ddim(get_named_beta_schedule("cosine", n3), eta=0.0)
                eng.ddim_sample_loop(x3, None, gt3, mask3, use_graph=True, out=out3)
                torch.cuda.synchronize()
            mem[name] = dict(max_memory_allocated_MB=torch.cuda.max_memory_allocated(dev) / 2 ** 20,
                             allocated_before_MB=base_alloc / 2 ** 20)
        eng._keep_loop = None
        mem["note"] = ("torch.cuda.max_memory_allocated during one loop call (torch allocations: tape, inputs, output); the "
                       "library's own workspaces come from cudaMalloc and are the same for both")
        mem["shape"] = "B=%d, T=%d, C=144, %d steps" % (B3, T, n3)
        res["memory_configs3"] = mem
    res["device"] = device_line(0)
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
