"""clock64 timeline of the fused feed-forward cluster kernel (M=1920: 120 CTAs) + mean launch time.
usage: python profiles/mlp_trace.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200.engine import Engine  # noqa: E402

eng = Engine("cuda:0")
g = torch.Generator().manual_seed(1)
M = 1920
x = torch.randn(M, 256, generator=g); w1 = torch.randn(1024, 256, generator=g) / 16; b1 = torch.randn(1024, generator=g) * 0.1
w2 = torch.randn(256, 1024, generator=g) / 32; b2 = torch.randn(256, generator=g) * 0.1; res = torch.randn(M, 256, generator=g)
# the MTRACE slots tc::mlp_tile writes (slot 0 = kernel entry), in clock64 cycles since entry
slots = {1: "barriers initialised", 2: "GEMM1 first operands landed", 3: "GEMM1 done", 5: "S written", 8: "GEMM2 done",
         9: "partials written", 10: "after cluster barrier", 11: "reduction stored", 12: "exit"}
tr = torch.zeros(256, 16, dtype=torch.int64, device="cuda")
eng.mlp(x, w1, b1, w2, b2, res, iters=3)
eng.mlp(x, w1, b1, w2, b2, res, iters=201, trace=tr)
print("fused feed-forward, M=%d: %.2f us/launch" % (M, eng.last_ms() * 1e3))
t = tr.cpu()[:120]
for i, n in slots.items():
    d = (t[:, i] - t[:, 0]).float()
    print("   %2d %-30s median %7.0f   max %7.0f" % (i, n, d.median().item(), d.max().item()))
