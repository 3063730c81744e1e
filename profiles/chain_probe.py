"""Timeline of the sampling step AS IT RUNS in the whole-loop graph (programmatic dependent launch on): every kernel
of the step marks %globaltimer at block entry, after its dependency wait and at block exit (idb_debug_chain_trace).
Per launch: its contribution to the chain (last exit - predecessor's last exit), split into the hand-off (predecessor's
last exit -> first block past griddepcontrol.wait) and the in-kernel critical path (-> last exit).
usage: python profiles/chain_probe.py [B] [steps] [graph mode: loop|step|off]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200 import synthetic as S  # noqa: E402
from interdiff_b200.diffusion.gaussian_diffusion import get_named_beta_schedule  # noqa: E402
from interdiff_b200.engine import Engine  # noqa: E402
from interdiff_b200.weights import bench_weights  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 12
mode = sys.argv[3] if len(sys.argv) > 3 else "loop"
NAMES = {1: "gemm", 2: "mlp_fused", 3: "k_qan_xattn_ln", 4: "k_attn_ln", 5: "k_xattn_ln", 6: "k_step_io"}

eng = Engine("cuda:0")
eng.load_denoiser(bench_weights("diffusion_smpl"), "smpl")
eng.init_diffusion(get_named_beta_schedule("cosine", steps))
b = S.make_smpl_batch(B=B, T=30)
eng.bind(b["cond"], 30)
tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps)).cuda()
gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
for _ in range(3):
    eng.p_sample_loop(tape, gt, mask, use_graph=mode)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    eng.p_sample_loop(tape, gt, mask, use_graph=mode)
e1.record()
torch.cuda.synchronize()
print("B=%d, %d-step loops, graph mode %s: %.1f us per step (probe off)" % (B, steps, mode, e0.elapsed_time(e1) / 5 / steps * 1e3))

CAP = 8192 * steps // 12 + 8192           # records per lane (64 lanes, lane = block & 63)
buf = torch.zeros(64, 2 + 2 * CAP, dtype=torch.int64, device="cuda")
buf[:, 1] = CAP
eng._chk(eng.lib.idb_debug_chain_trace(eng._h, buf.data_ptr()))
e0.record()
eng.p_sample_loop(tape, gt, mask, use_graph=mode)
e1.record()
torch.cuda.synchronize()
eng._chk(eng.lib.idb_debug_chain_trace(eng._h, None))
print("with the probe on: %.1f us per step" % (e0.elapsed_time(e1) / steps * 1e3))
h = buf.cpu().numpy().view(np.uint64)
assert int(h[:, 0].max()) <= CAP, "probe buffer too small"
key = np.concatenate([h[l, 2:2 + 2 * int(h[l, 0]):2] for l in range(64)])
t = np.concatenate([h[l, 3:3 + 2 * int(h[l, 0]):2] for l in range(64)]).astype(np.int64)
kind, ev = (key >> np.uint64(56)).astype(np.int64), ((key >> np.uint64(52)) & np.uint64(15)).astype(np.int64)
nb = ((key >> np.uint64(26)) & np.uint64(0x3FFFFFF)).astype(np.int64)
t0 = t.min()
t = t - t0

launches = []
for k in sorted(set(kind[kind > 0])):
    for g in sorted(set(nb[kind == k])):
        sel = (kind == k) & (nb == g)
        ent, ext = np.sort(t[sel & (ev == 0)]), np.sort(t[sel & (ev == 2)])
        assert len(ent) == len(ext) and len(ent) % g == 0, (k, g, len(ent), len(ext))
        for i in range(len(ent) // g):
            launches.append(dict(kind=int(k), grid=int(g), entry_min=int(ent[i * g]), entry_max=int(ent[(i + 1) * g - 1]),
                                 exit_min=int(ext[i * g]), exit_max=int(ext[(i + 1) * g - 1])))
launches.sort(key=lambda d: d["exit_max"])
waits = np.sort(t[ev == 1])
prev = None
for d in launches:
    lo = prev["exit_max"] if prev else -1
    w = waits[(waits > lo - 2000) & (waits <= d["exit_max"])]
    # dependency-wait marks of this launch: those after the predecessor's FIRST exit (a block passes the wait only when the
    # whole predecessor grid has completed; timer granularity leaves a little slack)
    w = w[w >= (prev["exit_min"] if prev else 0)]
    d["wait_min"] = int(w.min()) if len(w) else None
    d["wait_max"] = int(w.max()) if len(w) else None
    prev = d
per_step = len(launches) // steps
print("%d launches, %d per step; globaltimer resolution ~%d ns" % (len(launches), per_step, int(np.min(np.diff(np.unique(t))))))
# average the middle steps position by position
use = range(2, steps - 1)
print("%-3s %-16s %6s | %9s %9s %9s | %9s %9s %9s" % ("#", "kernel", "grid", "chain us", "handoff", "in-kernel", "early us", "last in", "exit spr"))
tot = 0.0
agg = {}
for pos in range(per_step):
    rows = []
    for s in use:
        i = s * per_step + pos
        d, p = launches[i], launches[i - 1]
        chain = d["exit_max"] - p["exit_max"]
        hand = (d["wait_min"] - p["exit_max"]) if d["wait_min"] is not None else float("nan")
        inker = (d["exit_max"] - d["wait_min"]) if d["wait_min"] is not None else float("nan")
        early = p["exit_max"] - d["entry_min"]          # how long before the predecessor's end the first block was resident
        # "last in": when the launch's LAST block entered, relative to the predecessor's last exit (blocks that only get an SM
        # when the predecessor's blocks leave it)
        rows.append((chain, hand, inker, early, d["entry_max"] - p["exit_max"], d["exit_max"] - d["exit_min"]))
    m = np.nanmean(np.array(rows, dtype=np.float64), axis=0) / 1e3
    d = launches[2 * per_step + pos]
    print("%-3d %-16s %6d | %9.2f %9.2f %9.2f | %9.2f %9.2f %9.2f" % (pos, NAMES.get(d["kind"], "?"), d["grid"], m[0], m[1], m[2], m[3], m[4], m[5]))
    tot += m[0]
    a = agg.setdefault((NAMES.get(d["kind"], "?"), d["grid"]), [0, 0.0, 0.0, 0.0])
    a[0] += 1; a[1] += m[0]; a[2] += m[1]; a[3] += m[2]
print("sum of chain contributions: %.1f us per step" % tot)
print("\nby kernel:  n  chain us (share)  hand-off  in-kernel")
for (name, g), a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print("  %-16s grid %4d  x%d  %7.1f (%4.1f %%)  %7.1f  %7.1f" % (name, g, a[0], a[1], 100 * a[1] / tot, a[2], a[3]))
