"""Accuracy / time trade-off of the fp32 promotion interval (k-blocks per tensor-core accumulation) of the wgmma GEMM."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200.engine import Engine  # noqa: E402

eng = Engine("cuda:0")
g = torch.Generator().manual_seed(0)
for (M, N, K) in ((1920, 1024, 256), (1920, 256, 256), (1920, 256, 1024)):
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    ref = A.double() @ W.double().T
    for nacc in (1, 2, 3, 5, 7):
        eng.lib.idb_debug_set_gemm_accumulators(nacc)
        out = eng.gemm(A, W).cpu().double()
        err = ((out - ref).abs().max() / ref.abs().max()).item()
        r = eng.gemm_microbench(M, N, K, iters=100, gelu=False)
        print("GEMM %dx%dx%d nacc<=%d: err %.2e  %.2f us/launch  %.1f TFLOP/s" % (M, N, K, nacc, err, r["ms"] * 1e3, 2.0 * M * N * K / r["ms"] / 1e9))
    eng.lib.idb_debug_set_gemm_accumulators(0)
eng.set_gemm_backend("simt")
for (M, N, K) in ((1920, 1024, 256), (1920, 256, 1024)):
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    ref = A.double() @ W.double().T
    err = ((eng.gemm(A, W).cpu().double() - ref).abs().max() / ref.abs().max()).item()
    print("SIMT fp32 %dx%dx%d: err %.2e" % (M, N, K, err))
