"""The persistent 64-column GEMM kernel: a CTA computes a run of column tiles of one or more row tiles, keeping the A row
block resident when K fits.  Its output must not depend on that schedule: every shape here is bit-identical to the same
kernel forced to one tile per CTA, writes one trace record per 128 x 64 tile, and meets the float64 bound of
tests/test_gpu_gemm_kernels.py."""
import math

import pytest
import torch

from tests.test_gpu_gemm_kernels import check, data, joined, split, tc_bound

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    from interdiff_b200.engine import Engine
    e = Engine(DEV)
    yield e
    e.lib.idb_debug_set_gemm_accumulators(911)
    e.close()


@pytest.fixture(autouse=True)
def _restore(eng):
    yield
    eng.lib.idb_debug_set_gemm_accumulators(911)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles(M, N):
    return ((M + 127) // 128) * ((N + 63) // 64)


def run(eng, A, W, M, N, persistent, **kw):
    """one GEMM on the persistent schedule or forced to one tile per CTA: (C, trace records written)"""
    eng.lib.idb_debug_set_gemm_accumulators(911 if persistent else 910)
    tr = torch.zeros(tiles(M, N) + 64, 16, dtype=torch.int64, device=DEV)
    out = kw.pop("out", None)
    if kw.get("split_k"):
        out = torch.zeros(M, N, device=DEV)
    out = eng.gemm(A, W, out=out, trace=tr, **kw)
    torch.cuda.synchronize()
    out = out.clone() if not isinstance(out, tuple) else tuple(o.clone() for o in out)
    return out, int((tr[:, 0] != 0).sum().item()), bool((tr[tiles(M, N):] == 0).all())


# (M, N, K, split_k): column tiles that do not divide over a row's CTAs, M and N tails, resident A (K = 152 and 256, the
# latter also with a row-tile count above the SM count), streamed A (K = 1024) with and without split-K
def shapes():
    big_m = (sms() + 2) * 128 - 40          # more row tiles than SMs: CTAs take further row tiles in turn
    return [(1920, 1300, 256, False), (1000, 1536, 152, False), (1920, 1100, 1024, False), (1920, 1024, 1024, True),
            (300, 660, 256, False), (big_m, 200, 152, False), (big_m, 136, 256, False)]


@pytest.mark.parametrize("case", range(7))
def test_schedule_independent_and_bounded(eng, record_property, case):
    M, N, K, split_k = shapes()[case]
    A, W = data("normal", (M, K), 3 * case + 1), data("normal", (N, K), 3 * case + 2) / math.sqrt(K)
    pA, pW = split(eng, A), split(eng, W)
    one, n_one, clean_one = run(eng, pA, pW, M, N, False, split_k=split_k)
    per, n_per, clean_per = run(eng, pA, pW, M, N, True, split_k=split_k)
    assert n_one == n_per == tiles(M, N) and clean_one and clean_per
    assert torch.equal(per, one), case
    A64, W64 = joined(pA), joined(pW)
    check(record_property, per, A64 @ W64.T, tc_bound(A64, W64, pA, pW, ksplit=2 if split_k else 1))


def test_epilogue_and_aux_zero_over_several_tiles_per_cta(eng):
    """bias, GELU, residual, fp32 and (hi, lo) outputs and the aux-zero side job on a shape where each CTA owns several
    column tiles: bit-identical to one tile per CTA, and the zeroed patch is exactly the requested matrix"""
    M, N, K, D = 1920, 1024, 256, 256
    A, W = data("normal", (M, K), 1), data("normal", (N, K), 2) / 16
    bias, res = data("normal", (N,), 3), data("normal", (M, N), 4)
    outs = []
    for persistent in (False, True):
        zb = torch.full((M + 10, D + 8), float("nan"), device=DEV)
        pair = (torch.empty(M, N, dtype=torch.float16, device=DEV), torch.empty(M, N, dtype=torch.float16, device=DEV))
        out, n, clean = run(eng, A, W, M, N, persistent, bias=bias, res=res, gelu=True, out=torch.empty(M, N, device=DEV),
                            out_pair=pair, zero=zb[:M, :D])
        assert n == tiles(M, N) and clean
        assert bool((zb[:M, :D] == 0).all()) and bool(torch.isnan(zb[M:]).all()) and bool(torch.isnan(zb[:, D:]).all())
        outs.append((out, pair[0].clone(), pair[1].clone()))
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a.view(torch.int16),
                           b.view(torch.int32) if b.dtype == torch.float32 else b.view(torch.int16))
