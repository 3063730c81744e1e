"""Time and error of the denoiser's GEMM shapes vs the number of k-blocks the wgmma GEMM accumulates in the tensor core
between two fp32 promotions (idb_debug_set_gemm_accumulators).
usage: python profiles/gemm_epi_probe.py"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200.engine import Engine  # noqa: E402

eng = Engine("cuda:0")
P = lambda t: C.c_void_p(t.data_ptr())
for (M, N, K, sk) in ((1920, 1024, 256, 0), (1920, 256, 1024, 1), (1920, 1536, 256, 0), (1920, 256, 256, 0)):
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") / K ** 0.5
    Ab, As, Wb, Ws = (torch.empty_like(t, dtype=torch.float16) for t in (A, A, W, W))
    eng._chk(eng.lib.idb_debug_split(eng._h, P(A), P(Ab), P(As), M, K, K, eng._stream()))
    eng._chk(eng.lib.idb_debug_split(eng._h, P(W), P(Wb), P(Ws), N, K, K, eng._stream()))
    ref = A.double().cpu() @ W.double().cpu().T
    for nacc in (1, 2, 3, 4, 7):
        eng.lib.idb_debug_set_gemm_accumulators(nacc)
        out = torch.zeros(M, N, device="cuda")
        run = lambda it: eng._chk(eng.lib.idb_debug_gemm_presplit(eng._h, P(Ab), P(As), P(Wb), P(Ws), None, P(out), M, N, K,
                                                                  128 if sk else 0, it, None, eng._stream()))
        run(1)
        torch.cuda.synchronize()
        err = ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()
        run(5)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(300); e1.record()
        torch.cuda.synchronize()
        print("%dx%dx%d%s nacc<=%d: %.2f us/launch  err %.2e" % (M, N, K, " split-K 2" if sk else "", nacc, e0.elapsed_time(e1) / 300 * 1e3, err))
eng.lib.idb_debug_set_gemm_accumulators(0)
