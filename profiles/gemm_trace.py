"""Per-CTA clock64 timeline + timing of the wgmma GEMM pipeline on PRE-SPLIT operands (the path the
denoiser uses) -- debug aid."""
import ctypes as C
import itertools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200.engine import Engine  # noqa: E402

eng = Engine("cuda:0")
P = lambda t: C.c_void_p(t.data_ptr())
names = ["entry", "setup_done", "tma_first_issued", "tma_all_issued", "conv_first_full", "conv_first_done", "mma_first_ready",
         "mma_all_issued", "conv_all_done", "epi_acc_ready", "epi_done", "final_sync", "dealloc"]
show = ("setup_done", "tma_first_issued", "tma_all_issued", "mma_first_ready", "mma_all_issued", "epi_acc_ready", "epi_done", "dealloc")
shapes = ((1920, 1024, 256), (1920, 256, 1024), (1920, 256, 256), (1920, 1536, 256), (1920, 256, 152), (1920, 144, 256))   # .., QKV', embedding, heads
for (M, N, K), flags in itertools.product(shapes, (0, 64)):
    if flags and N != 1024:
        continue
    eng.lib.idb_debug_set_gemm_accumulators(1000 + flags)
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") / K ** 0.5
    Ab, As, Wb, Ws = (torch.empty_like(t, dtype=torch.float16) for t in (A, A, W, W))
    eng._chk(eng.lib.idb_debug_split(eng._h, P(A), P(Ab), P(As), M, K, K, eng._stream()))
    eng._chk(eng.lib.idb_debug_split(eng._h, P(W), P(Wb), P(Ws), N, K, K, eng._stream()))
    out = torch.empty(M, N, device="cuda")
    tr = torch.zeros(4096, 16, dtype=torch.int64, device="cuda")
    run = lambda it, trace: eng._chk(eng.lib.idb_debug_gemm_presplit(eng._h, P(Ab), P(As), P(Wb), P(Ws), None, P(out), M, N, K, 0, it,
                                                                     P(tr) if trace else None, eng._stream()))
    run(3, False)
    run(1, True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); run(200, False); e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 200 * 1e3
    if flags == 0:
        err = ((out.double().cpu() - A.double().cpu() @ W.double().cpu().T).abs().max() / (A.double().cpu() @ W.double().cpu().T).abs().max()).item()
    t = tr.cpu()
    ncta = int((t[:, 0] != 0).sum())
    t = t[:ncta]
    print("PRE GEMM %dx%dx%d flags=%d: %d CTAs, %.2f us/launch (%.1f TFLOP/s)%s" % (
        M, N, K, flags, ncta, us, 2.0 * M * N * K / us / 1e6, ("  err %.2e" % err) if flags == 0 else "  (big x big MMA only)"))
    for i, n in enumerate(names):
        if n in show:
            d = (t[:, i] - t[:, 0]).float()
            print("   %-18s median %8.0f   max %8.0f" % (n, d.median().item(), d.max().item()))
