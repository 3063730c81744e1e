"""Per-tile clock64 timeline + timing of the wgmma GEMM pipeline on PRE-SPLIT operands (the path the
denoiser uses) -- debug aid.

Trace record per 128 x 64 output tile (slot: what thread 0 / the producer's lane 0 wrote there):
  0 tile start (the CTA's first tile: kernel entry)      1 barriers set up (the CTA's first tile only)
  2 producer: first loads issued past the dependency wait 3 producer: every load of the CTA issued
  6 first full stage of the tile                          9 last MMA of the tile retired
 10 epilogue stores issued                               11 CTA exit (the CTA's last tile only)
 12 CTA entry, in the record that holds slot 11 when that record is not the CTA's first tile
clock64 is per SM, so only differences inside one record are printed."""
import ctypes as C
import itertools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interdiff_b200.engine import Engine  # noqa: E402

eng = Engine("cuda:0")
P = lambda t: C.c_void_p(t.data_ptr())
SMS = torch.cuda.get_device_properties(0).multi_processor_count


def l2_bytes(M, N, K, ctas):
    """L2 -> SM bytes of one launch from the tile shape: fp16 hi + lo of every 128 x 64 A box and 64 x 64 W box loaded
    (TMA boxes are whole, K rounded up to 64).  A is loaded once per tile, or once per (CTA, row tile) when fewer CTAs
    than tiles ran and the whole K fits in shared memory."""
    rt, ct, kp = (M + 127) // 128, (N + 63) // 64, (K + 63) // 64 * 64
    a_loads = rt * max(1, ctas // rt) if (ctas < rt * ct and kp <= 256) else rt * ct
    return a_loads * 128 * kp * 4, rt * ct * 64 * kp * 4


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
    t = t[t[:, 0] != 0]
    first = t[t[:, 1] != 0]
    last = t[t[:, 11] != 0]
    ctas = len(first)
    a_b, w_b = l2_bytes(M, N, K, ctas)
    print("PRE GEMM %dx%dx%d flags=%d: %d tiles on %d CTAs, %.2f us/launch (%.1f TFLOP/s)%s" % (
        M, N, K, flags, len(t), ctas, us, 2.0 * M * N * K / us / 1e6, ("  err %.2e" % err) if flags == 0 else "  (big x big MMA only)"))
    print("   L2 -> SM per launch: %.1f MB (A %.1f MB, W %.1f MB)" % ((a_b + w_b) / 1e6, a_b / 1e6, w_b / 1e6))

    def row(name, d):
        d = d.float()
        print("   %-32s median %8.0f   max %8.0f   sum/CTA %8.0f" % (name, d.median().item(), d.max().item(), d.sum().item() / ctas))
    row("CTA entry -> first full stage", first[:, 6] - first[:, 0])
    row("producer: first loads issued", first[:, 2] - first[:, 0])
    row("tile start -> first full stage", t[:, 6] - t[:, 0])
    row("MMA span (first full -> retired)", t[:, 9] - t[:, 6])
    row("epilogue span", t[:, 10] - t[:, 9])
    entry = torch.where(last[:, 12] != 0, last[:, 12], last[:, 0])
    row("CTA entry -> exit", last[:, 11] - entry)
