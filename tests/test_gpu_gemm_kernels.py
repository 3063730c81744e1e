"""Kernel-level tests of every wgmma GEMM variant and of the fused feed-forward kernel, element by element against float64
references computed on the device.

Error model of the tensor path (gemm_wgmma.cu), per output element, u = 2^-24 (fp32 unit roundoff):

* Operands.  x is carried as hi = fp16_rn(x), lo = fp16_rn((x - hi) 2^11).  When lo is a normal fp16 number the pair
  represents x to 2^-23 |x| (lo has 11 bits and its sign gives one more).  lo is subnormal when |x - hi| < 2^-25; its spacing is
  then 2^-24, i.e. 2^-35 in units of x, so  |x - x^| <= rho(x) = max(2^-23 |x|, 2^-36).  A product of two represented
  factors is off by rho(a)|w| + |a|rho(w) (plus a 2^-46 |a||w| cross term, covered below).
* Dropped lo*lo.  The kernel forms hi*hi + 2^-11 (lo*hi + hi*lo); the missing 2^-22 lo*lo is at most
  sigma(a) sigma(w) with sigma(x) = (1 + 2^-10) max(2^-11 |x|, 2^-25) >= |x - hi|.
* Tensor-core accumulation.  One wgmma k-step adds 16 exact fp16 products to an fp32 accumulator and truncates the sum to
  fp32.  Model: at most 2 ulp per instruction (one for the alignment of the 17 addends, one for the final truncation), i.e.
  4u times the running sum of |a||w| through that k-step.  With the per-k-block promotion the main accumulator restarts at
  every k-block of 64 (4 k-steps), so the product at k-step t (0..3) of its block enters 4 - t such sums: weight 4 (4 - t).
  With single_acc the accumulator runs over all K/16 k-steps: weight 4 (K/16 - s) for global k-step s.
* The small accumulator (lo*hi + hi*lo, 2 instructions per k-step, |terms| <= 2.01 |a||w|) never restarts; it is scaled by
  2^-11 in the epilogue: weight 2^-11 * 2 * 4 * 2.01 (K/16 - s) < (K/16 - s) / 127.
* Promotion.  sum += part is one round-to-nearest fp32 addition per k-block (u times the running sum); the first is
  exact (sum = 0), so a product in k-block b (0-based, nb blocks) enters nb - max(b, 1) of them.  Split-K counts blocks per
  half and adds one rounding (u) for the reduction of the two halves onto the zeroed C.
* Epilogue.  fmaf(small, 2^-11, sum): 1u.  Bias and residual additions: u times the magnitude after each addition.

Summing the weights over k gives the bound as  u |A| diag(omega) |W|^T + u (rho and sigma terms), which is at most
c u (|A||W|^T) with c = 8.02 + 16 + (K/64 - 1) + K/2032 + 1 for promoted GEMMs (58.0 at K = 2048) - the per-k weights make
it tighter where the error cannot reach.  For single_acc, c = 8.02 + K/4 + K/2032 + 1.  The SIMT backend runs one fmaf chain
per element: the plain gamma_K = K u / (1 - K u).

The bound is a worst case.  On one-signed data every truncation points the same way, so an accumulator that is not
promoted fails it at K = 4096 (test_bound_detects_missing_promotion), as does the kernel without its lo terms
(test_bound_detects_dropped_lo_terms).  Each case records its largest err / bound as the `ratio` property.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    from interdiff_b200.engine import Engine
    e = Engine(DEV)
    yield e
    e.lib.idb_debug_set_gemm_accumulators(0)
    e.lib.idb_debug_set_gemm_accumulators(901)
    e.close()


@pytest.fixture(autouse=True)
def _restore(eng):
    yield
    eng.set_gemm_backend("tcgen05")
    eng.set_gemm_multicast(True)
    eng.lib.idb_debug_set_gemm_accumulators(0)
    eng.lib.idb_debug_set_gemm_accumulators(901)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------ operand helpers
def split(eng, x, ld=None):
    """fp16 (hi, lo) pair of an fp32 device matrix via the library's split (views [rows, cols] of [rows, ld] buffers)"""
    x = x.to(DEV, torch.float32).contiguous()
    rows, cols = x.shape
    ld = ld or cols
    hi = torch.zeros(rows, ld, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi)
    eng._chk(eng.lib.idb_debug_split(eng._h, eng._ptr(x), eng._ptr(hi), eng._ptr(lo), rows, cols, ld, eng._stream()))
    return hi[:, :cols], lo[:, :cols]


def joined(p):
    """the value a pair represents, exactly (float64)"""
    return p[0].double() + p[1].double() * 2.0 ** -11


def rho(x):
    return torch.clamp(x.abs() * 2.0 ** -23, min=2.0 ** -36)


def sigma(x):
    return (1 + 2.0 ** -10) * torch.clamp(x.abs() * 2.0 ** -11, min=2.0 ** -25)


def kstep_weights(K, single_acc=False, ksplit=1):
    """omega_k of the module docstring (without the operand terms), float64 on the device"""
    nkb = (K + 63) // 64
    k = torch.arange(K, device=DEV)
    b, t = k // 64, (k % 64) // 16
    if ksplit == 2 and nkb >= 2:
        per = (nkb + 1) // 2
        half = b // per
        lb = b - half * per
        nb = torch.where(half == 0, torch.full_like(b, per), torch.full_like(b, nkb - per))
        nsteps = nb * 4
        s = lb * 4 + t
        extra = 1.0                           # the reduction of the two halves
    else:
        lb, nb, nsteps, s, extra = b, torch.full_like(b, nkb), torch.full_like(b, nkb * 4), b * 4 + t, 0.0
    small = (nsteps - s).double() / 127.0
    if single_acc:
        trunc, prom = 4.0 * (nsteps - s).double(), torch.zeros(K, device=DEV, dtype=torch.float64)
    else:
        trunc, prom = 4.0 * (4 - t).double(), (nb - torch.clamp(lb, min=1)).double()
    return trunc + prom + small + 1.0 + extra


def tc_bound(A, W, pairA=None, pairW=None, single_acc=False, ksplit=1):
    """element-wise bound (float64 [M, N]) on |C - A W^T| of the tensor path, before bias / activation / residual.
    A, W: float64 exact operands; pairA / pairW given: the operands already are pairs (no representation error)."""
    K = A.shape[1]
    om = kstep_weights(K, single_acc, ksplit)
    aA, aW = A.abs(), W.abs()
    b = U * ((aA * om) @ aW.T)
    b += sigma(A) @ sigma(W).T
    if pairA is None:
        b += rho(A) @ aW.T
    if pairW is None:
        b += aA @ rho(W).T
    b += 2.0 ** -46 * (aA @ aW.T)
    return b


def simt_bound(A, W):
    K = A.shape[1]
    return (K * U / (1 - K * U)) * (A.abs() @ W.abs().T)


def epilogue(y, e, bias=None, res=None, gelu=False, silu=False):
    """exact epilogue on y (float64) and the bound e (on y) carried through it: each fp32 addition adds u |result|,
    GELU / SiLU have slope <= 1.13 / 1.10 and their own error (common.cuh: erf to 1.0e-7 -> 2.5e-7 max(|x|, 1) for GELU;
    SiLU x / (1 + expf(-x)): 6u relative (expf 2 ulp, the addition and the division), plus 1e-36 absolute where expf overflows (x < -88.7, |silu| < 3e-37))"""
    if bias is not None:
        y = y + bias.double()
        e = e + U * y.abs()
    if gelu:
        e = 1.13 * e + 2.5e-7 * torch.clamp(y.abs(), min=1.0)
        y = torch.nn.functional.gelu(y)
    if silu:
        e = 1.10 * e + 6 * U * (y * torch.sigmoid(y)).abs() + 1e-36
        y = y * torch.sigmoid(y)
    if res is not None:
        y = y + res.double()
        e = e + U * y.abs()
    return y, e


def check(record_property, got, want, bound, tag=""):
    err = (got.double() - want).abs()
    ratio = (err / bound).max().item()
    record_property("ratio" + tag, ratio)
    assert torch.isfinite(got).all()
    assert ratio <= 1.0, (tag, ratio)
    return ratio


def data(family, shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if family == "normal":
        return torch.randn(*shape, generator=g, device=DEV)
    return torch.rand(*shape, generator=g, device=DEV)


# ------------------------------------------------------------------ 1. element-wise bound, both backends, two families
BOUND_CASES = [("normal", 1920, 1536, 256), ("normal", 300, 260, 1024), ("normal", 129, 200, 4096),
               ("uniform", 1920, 256, 1024), ("uniform", 257, 132, 4096), ("uniform", 65, 68, 200)]


@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
@pytest.mark.parametrize("family,M,N,K", BOUND_CASES)
def test_elementwise_bound(eng, record_property, backend, family, M, N, K):
    eng.set_gemm_backend(backend)
    A, W = data(family, (M, K), M + K), data(family, (N, K), N + 7 * K)
    bias, res = data(family, (N,), 3), data(family, (M, N), 4)
    A64, W64 = A.double(), W.double()
    y = A64 @ W64.T
    bnd = simt_bound(A64, W64) if backend == "simt" else tc_bound(A64, W64)
    check(record_property, eng.gemm(A, W), y, bnd, "_plain")
    want, e = epilogue(y, bnd, bias=bias, res=res)
    check(record_property, eng.gemm(A, W, bias=bias, res=res), want, e, "_bias_res")


def test_bound_detects_missing_promotion(eng, record_property):
    """one tensor-core accumulator over K = 4096 of one-signed data (promotion every 512 k-blocks, i.e. never): the
    truncations add up linearly in K and the promoted kernel's bound must fail."""
    A, W = data("uniform", (257, 4096), 1), data("uniform", (132, 4096), 2)
    y = A.double() @ W.double().T
    bnd = tc_bound(A.double(), W.double())
    eng.set_gemm_backend("tcgen05")
    ok = check(record_property, eng.gemm(A, W), y, bnd, "_promoted")
    eng.lib.idb_debug_set_gemm_accumulators(512)
    bad = ((eng.gemm(A, W).double() - y).abs() / bnd).max().item()
    record_property("ratio_unpromoted", bad)
    assert bad > 1.0, (ok, bad)


def test_bound_detects_dropped_lo_terms(eng, record_property):
    A, W = data("uniform", (257, 1024), 5), data("normal", (132, 1024), 6)
    y = A.double() @ W.double().T
    bnd = tc_bound(A.double(), W.double())
    eng.set_gemm_backend("tcgen05")
    bad = ((eng.gemm(A, W, hi_only=True).double() - y).abs() / bnd).max().item()
    record_property("ratio_hi_only", bad)
    assert bad > 1.0


# ------------------------------------------------------------------ 3. edge shapes of the tensor path
EDGE_M = [1, 63, 64, 65, 127, 128, 129, 257, 1920]
EDGE_N = [8, 12, 60, 64, 68, 124, 132, 1536]
EDGE_K = [8, 12, 36, 60, 64, 68, 200, 1024, 4096]
# every value of each list at least once, cycled against the others (no full product)
EDGE = [(EDGE_M[i % 9], EDGE_N[(i * 5) % 8], EDGE_K[(i * 4) % 9]) for i in range(18)]


@pytest.mark.parametrize("M,N,K", EDGE)
def test_edge_shapes(eng, record_property, M, N, K):
    A, W = data("normal", (M, K), M * 3 + K), data("normal", (N, K), N * 5 + K) / math.sqrt(K)
    y = A.double() @ W.double().T
    out, ctas = traced(eng, A, W)
    assert ctas == ((N + 63) // 64) * ((M + 127) // 128)          # the tensor path ran (64-column tiles)
    check(record_property, out, y, tc_bound(A.double(), W.double()))
    # the same operands as pre-split pairs (row stride rounded up to 8 elements, as TMA needs)
    ld = (K + 7) // 8 * 8
    pA, pW = split(eng, A, ld), split(eng, W, ld)
    y2 = joined(pA) @ joined(pW).T
    out, ctas = traced(eng, pA, pW)
    assert ctas == ((N + 63) // 64) * ((M + 127) // 128)
    check(record_property, out, y2, tc_bound(joined(pA), joined(pW), pA, pW), "_pairs")


# ------------------------------------------------------------------ 4. 128-column and multicast-pair kernels
def wide_shapes():
    out = []
    for rt in (3, 5):
        n128 = -(-sms() // (2 * rt))           # 2 * row_tiles * column tiles >= SMs: the 128-column kernels are chosen
        for tail in (4, 64):
            out.append(((rt - 1) * 128 + 1 + (rt == 3) * 64, (n128 - 1) * 128 + tail, 200))
    return out


def traced(eng, A, W, **kw):
    """GEMM with the per-CTA timeline on: returns (C, number of CTAs that wrote their entry slot)"""
    M, N = len(A[0]) if isinstance(A, tuple) else A.shape[0], len(W[0]) if isinstance(W, tuple) else W.shape[0]
    tr = torch.zeros(((N + 63) // 64) * (((M + 127) // 128) + 1), 16, dtype=torch.int64, device=DEV)
    out = eng.gemm(A, W, trace=tr, **kw)
    torch.cuda.synchronize()
    return out, int((tr[:, 0] != 0).sum().item())


@pytest.mark.parametrize("case", range(4))
def test_wide_and_multicast_kernels(eng, record_property, case):
    M, N, K = wide_shapes()[case]
    rt, n64, n128 = (M + 127) // 128, (N + 63) // 64, (N + 127) // 128
    assert rt % 2 == 1 and N % 128 in (4, 64) and K % 64
    A, W = data("normal", (M, K), case), data("normal", (N, K), case + 10) / math.sqrt(K)
    mc, ctas_mc = traced(eng, A, W, single_acc=True)
    eng.set_gemm_multicast(False)
    wide, ctas_wide = traced(eng, A, W, single_acc=True)
    eng.lib.idb_debug_set_gemm_accumulators(900)
    narrow, ctas_narrow = traced(eng, A, W, single_acc=True)
    record_property("grids", (ctas_mc, ctas_wide, ctas_narrow))
    assert ctas_mc == n128 * (rt + 1)        # multicast pairs: an even number of row tiles, the last one empty
    assert ctas_wide == n128 * rt
    assert ctas_narrow == n64 * rt
    assert torch.equal(mc, wide) and torch.equal(mc, narrow)
    y = A.double() @ W.double().T
    check(record_property, mc, y, tc_bound(A.double(), W.double(), single_acc=True))


def test_default_gemm_takes_64_column_tiles(eng):
    """promoted GEMMs never take the 128-column kernel, whatever their size"""
    A, W = data("normal", (1920, 256), 1), data("normal", (1536, 256), 2)
    _, ctas = traced(eng, A, W)
    assert ctas == 24 * 15


# ------------------------------------------------------------------ 5. epilogue and outputs
@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
def test_pair_output_equals_split_of_fp32_output(eng, backend):
    eng.set_gemm_backend(backend)
    M, N, K = 200, 132, 96
    A, W = data("normal", (M, K), 1), data("normal", (N, K), 2) / 8
    bias, res = data("normal", (N,), 3), data("normal", (M, N), 4)
    for bits in range(16):
        if bits & 2 and bits & 8:
            continue                                           # GELU and SiLU are alternatives
        kw = dict(bias=bias if bits & 1 else None, res=res if bits & 4 else None, gelu=bool(bits & 2), silu=bool(bits & 8))
        pair = (torch.empty(M, N, dtype=torch.float16, device=DEV), torch.empty(M, N, dtype=torch.float16, device=DEV))
        out = eng.gemm(A, W, out=torch.empty(M, N, device=DEV), out_pair=pair, **kw)
        want = split(eng, out)
        assert torch.equal(pair[0].view(torch.int16), want[0].view(torch.int16)), bits
        assert torch.equal(pair[1].view(torch.int16), want[1].view(torch.int16)), bits
        only = (torch.empty(M, N, dtype=torch.float16, device=DEV), torch.empty(M, N, dtype=torch.float16, device=DEV))
        eng.gemm(A, W, out_pair=only, **kw)                    # split-only output (C = NULL), as ff1 runs
        assert torch.equal(only[0].view(torch.int16), want[0].view(torch.int16)), bits
        assert torch.equal(only[1].view(torch.int16), want[1].view(torch.int16)), bits


@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
@pytest.mark.parametrize("act", ["gelu", "silu"])
def test_activation_accuracy_on_a_grid(eng, record_property, backend, act):
    """GELU / SiLU epilogue on every multiple of 2^-10 in [-8, 8] plus large arguments of both signs (exact in the pairs):
    the 'GEMM' multiplies by the identity, so only the activation's error remains"""
    eng.set_gemm_backend(backend)
    x = torch.arange(-8 * 1024, 8 * 1024 + 1, dtype=torch.float64) / 1024.0
    big = torch.tensor([-60000.0, -1000.0, -104.0, -100.0, -89.0, -88.5, -87.0, -50.0, -20.0, -12.0, 12.0, 20.0, 100.0, 60000.0],
                       dtype=torch.float64)
    x = torch.cat([x, big])
    x = x[: (x.numel() // 8) * 8].reshape(-1, 8).to(DEV)
    out = eng.gemm(x.float(), torch.eye(8, device=DEV), **{act: True}).double()
    want, e = epilogue(x, torch.zeros_like(x), **{act: True})
    check(record_property, out, want, e + 2 * U * want.abs())   # + the fp32 rounding of the result


# ------------------------------------------------------------------ 6. strides, NaN padding, sentinel outputs
SENT = -7.777e33


@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
@pytest.mark.parametrize("presplit", [False, True])
def test_strides_padding_and_untouched_outputs(eng, record_property, backend, presplit):
    eng.set_gemm_backend(backend)
    M, N, K = 130, 68, 200
    lda, ldw, ldr, ldc = 264, 232, 76, 80
    A, W = data("normal", (M, K), 1), data("normal", (N, K), 2) / 14
    bias, res = data("normal", (N,), 3), data("normal", (M, N), 4)
    nan = float("nan")
    if presplit:
        pA, pW = split(eng, A, lda), split(eng, W, ldw)
        for p, k in ((pA, K), (pW, K)):
            for part in p:
                part.as_strided((part.shape[0], part.stride(0) - k), (part.stride(0), 1), part.storage_offset() + k).fill_(nan)
        opA, opW = pA, pW
        A64, W64 = joined(pA), joined(pW)
    else:
        Ab = torch.full((M, lda), nan, device=DEV); Ab[:, :K] = A
        Wb = torch.full((N, ldw), nan, device=DEV); Wb[:, :K] = W
        opA, opW = Ab[:, :K], Wb[:, :K]
        A64, W64 = A.double(), W.double()
    Rb = torch.full((M, ldr), nan, device=DEV); Rb[:, :N] = res
    Cb = torch.full((M + 70, ldc), SENT, device=DEV)
    hb = torch.full((M + 70, ldc), -1234.0, dtype=torch.float16, device=DEV)
    lb = torch.full_like(hb, 4320.0)
    out = eng.gemm(opA, opW, bias=bias, res=Rb[:, :N], out=Cb[:M, :N], out_pair=(hb[:M, :N], lb[:M, :N]))
    y = A64 @ W64.T
    bnd = simt_bound(A64, W64) if backend == "simt" else tc_bound(A64, W64, *((opA, opW) if presplit else (None, None)))
    want, e = epilogue(y, bnd, bias=bias, res=res)
    check(record_property, out, want, e)
    mask = torch.ones(M + 70, ldc, dtype=torch.bool, device=DEV)
    mask[:M, :N] = False
    assert bool((Cb[mask] == SENT).all())
    assert bool((hb[mask] == -1234.0).all()) and bool((lb[mask] == 4320.0).all())
    want_pair = split(eng, Cb[:M, :N])
    assert torch.equal(hb[:M, :N], want_pair[0]) and torch.equal(lb[:M, :N], want_pair[1])


# ------------------------------------------------------------------ 7. aux zero + split-K, as ff1 / ff2 pair them
@pytest.mark.parametrize("wide", [False, True])
def test_aux_zero_then_split_k(eng, record_property, wide):
    D = 256
    if wide:     # a single-accumulator producer with 16 128-column tiles x 5 row tiles (>= the SMs of any H100 / 2)
        M, F = 640, 2048
    else:
        M, F = 300, 1024
    x, w1 = data("normal", (M, D), 1), data("normal", (F, D), 2) / 16
    zb = torch.full((M + 50, D + 40), float("nan"), device=DEV)
    hid = (torch.empty(M, F, dtype=torch.float16, device=DEV), torch.empty(M, F, dtype=torch.float16, device=DEV))
    tr = torch.zeros(((F + 63) // 64) * ((M + 127) // 128), 16, dtype=torch.int64, device=DEV)
    eng.gemm(split(eng, x), split(eng, w1), gelu=True, out_pair=hid, zero=zb[:M, :D], single_acc=wide, pdl=True, trace=tr)
    torch.cuda.synchronize()
    ctas = int((tr[:, 0] != 0).sum().item())
    assert ctas == ((F + 127) // 128 if wide else (F + 63) // 64) * ((M + 127) // 128)
    assert bool((zb[:M, :D] == 0).all())
    assert bool(torch.isnan(zb[M:]).all()) and bool(torch.isnan(zb[:, D:]).all())
    # consumer: split-K onto the cleared rows (row stride D + 40), twice for bit-reproducibility
    w2, b2, r = data("normal", (D, F), 3) / 32, data("normal", (D,), 4), data("normal", (M, D), 5)
    pw2 = split(eng, w2)
    outs = [eng.gemm(hid, pw2, bias=b2, res=r, split_k=True, out=zb[:M, :D], pdl=True).clone()]
    zb[:M, :D] = 0
    outs.append(eng.gemm(hid, pw2, bias=b2, res=r, split_k=True, out=zb[:M, :D], pdl=True).clone())
    assert torch.equal(outs[0], outs[1])
    H, W2 = joined(hid), joined(pw2)
    y = H @ W2.T
    want, e = epilogue(y, tc_bound(H, W2, hid, pw2, ksplit=2), bias=b2, res=r)
    # bias and residual are added to the leading half's partial sum, whose magnitude is bounded by |H||W2|^T, not by |y|
    e = e + 2 * U * (H.abs() @ W2.abs().T + b2.double().abs() + r.double().abs())
    check(record_property, outs[0], want, e)


def test_aux_zero_columns_must_split_over_tiles(eng):
    from interdiff_b200.engine import EngineError
    x, w = data("normal", (64, 64), 1), data("normal", (256, 64), 2)
    zb = torch.zeros(64, 256, device=DEV)
    with pytest.raises(EngineError, match="aux zero"):
        eng.gemm(x, w, zero=zb[:, :100])         # 4 column tiles of 64: 100 columns are not 4 x a multiple of 4


# ------------------------------------------------------------------ 8. row-slice invariance
SLICES = [(100, 300), (127, 129), (0, 1), (255, 900)]


@pytest.mark.parametrize("mode", ["narrow", "split_k", "single_acc"])
def test_row_slices_are_bit_identical(eng, mode):
    if mode == "single_acc":
        M, N, K = 1920, -(-sms() // 30) * 128 + 64, 200
    else:
        M, N, K = 1920, 256, 1024
    A, W = data("normal", (M, K), 1), data("normal", (N, K), 2) / 32
    pA, pW = split(eng, A), split(eng, W)
    kw = dict(split_k=mode == "split_k", single_acc=mode == "single_acc")
    full = eng.gemm(pA, pW, **kw)
    for r0, r1 in SLICES:
        part = eng.gemm((pA[0][r0:r1], pA[1][r0:r1]), pW, **kw)
        assert torch.equal(part, full[r0:r1]), (mode, r0, r1)
        part = eng.gemm(A[r0:r1], W, **kw)
        assert torch.equal(part, full[r0:r1]), (mode, r0, r1, "fp32")


def test_feed_forward_row_slices_are_bit_identical(eng):
    x, w1, b1, w2, b2, res = mlp_data(1920, 1)
    full = eng.mlp(x, w1, b1, w2, b2, res)
    for r0, r1 in SLICES:
        assert torch.equal(eng.mlp(x[r0:r1], w1, b1, w2, b2, res[r0:r1]), full[r0:r1]), (r0, r1)


# ------------------------------------------------------------------ 9. operand domain
def test_operand_domain(eng, record_property):
    """rows of A scaled by 2^e, e in [-14, 15], and entries of exactly +-65504: the bound with the 2^-36 floor of the
    module docstring holds.  Rows at e in [-24, -15] (hi subnormal) are checked against the same bound and their error
    relative to |A||W|^T is recorded."""
    K, N = 256, 64
    es = list(range(-24, 16))
    g = torch.Generator(device=DEV).manual_seed(9)
    A = (torch.rand(len(es) + 2, K, generator=g, device=DEV) * 2 - 1)
    A[: len(es)] *= torch.tensor([2.0 ** e for e in es], device=DEV)[:, None]
    A[len(es)] = 65504.0
    A[len(es) + 1, ::2], A[len(es) + 1, 1::2] = -65504.0, 65504.0
    W = torch.rand(N, K, generator=g, device=DEV) * 2 - 1
    y = A.double() @ W.double().T
    out = eng.gemm(A, W).double()
    bnd = tc_bound(A.double(), W.double())
    check(record_property, out, y, bnd)
    rel = ((out - y).abs() / (A.double().abs() @ W.double().abs().T)).max(dim=1).values
    for i, e in enumerate(es):
        record_property("rel_err_2^%d" % e, rel[i].item())


# ------------------------------------------------------------------ 10. feed-forward kernel
def mlp_data(M, seed, xscale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, 256, generator=g, device=DEV) * xscale
    w1 = torch.randn(1024, 256, generator=g, device=DEV) / 16
    b1 = torch.randn(1024, generator=g, device=DEV) * 0.1
    w2 = torch.randn(256, 1024, generator=g, device=DEV) / 32
    b2 = torch.randn(256, generator=g, device=DEV) * 0.1
    res = torch.randn(M, 256, generator=g, device=DEV)
    return x, w1, b1, w2, b2, res


def mlp_reference(x, w1, b1, w2, b2, res):
    """float64 output and its element-wise bound.  GEMM 1 (K = 256) and each of GEMM 2's four partials (K = 256 of the
    hidden layer) run on one tensor-core accumulator (single_acc weights); GEMM 2's truncation weight is bounded by its
    largest (16 k-steps) because the k order inside a partial depends on the CTA; the four partials are summed in fp32
    (3u of their magnitude), then bias and residual (u each)."""
    X, W1, W2 = x.double(), w1.double(), w2.double()
    v = X @ W1.T + b1.double()
    e1 = tc_bound(X, W1, single_acc=True) + U * v.abs()
    h = torch.nn.functional.gelu(v)
    eh = 1.13 * e1 + 2.5e-7 * torch.clamp(v.abs(), min=1.0) + rho(h)          # + the split of h into its pair
    P2 = h.abs() @ W2.abs().T
    e2 = eh @ W2.abs().T + U * (64 + 1 / 127 * 16 + 1 + 3) * P2 + sigma(h) @ sigma(W2).T + h.abs() @ rho(W2).T
    z = h @ W2.T + b2.double()
    e2 = e2 + U * z.abs()
    z = z + res.double()
    return z, e2 + U * z.abs()


def layer_norm_reference(z, ez, lw, lb):
    """float64 LayerNorm and a first-order bound from the input bound ez and the kernel's fp32 two-pass statistics (mean and
    centred sum of squares over 256 values: <= 8u of max|z| for the mean, then the centring subtraction)"""
    mu = z.mean(dim=1, keepdim=True)
    c = z - mu
    sd = torch.sqrt((c * c).mean(dim=1, keepdim=True) + 1e-5)
    E = ez.max(dim=1, keepdim=True).values + 8 * U * z.abs().max(dim=1, keepdim=True).values
    y = c / sd * lw.double() + lb.double()
    e = lw.double().abs() / sd * (ez + E + U * c.abs() + c.abs() / sd * 2 * (E + 8 * U * sd)) + 4 * U * y.abs()
    return y, e


@pytest.mark.parametrize("M", [1, 5, 129, 1920])
@pytest.mark.parametrize("norm", [False, True])
def test_feed_forward_outputs(eng, record_property, M, norm):
    x, w1, b1, w2, b2, res = mlp_data(M, M)
    g = torch.Generator(device=DEV).manual_seed(M + 100)
    lw, lb = (1 + 0.1 * torch.randn(256, generator=g, device=DEV), 0.1 * torch.randn(256, generator=g, device=DEV)) if norm else (None, None)
    out = torch.full((M + 130, 256), SENT, device=DEV)
    zh = torch.full((M + 130, 256), -1234.0, dtype=torch.float16, device=DEV)
    zl = torch.full_like(zh, 4320.0)
    eng.mlp(x, w1, b1, w2, b2, res, ln_w=lw, ln_b=lb, out=out, out_pair=(zh, zl))
    assert bool((out[M:] == SENT).all()) and bool((zh[M:] == -1234.0).all()) and bool((zl[M:] == 4320.0).all())
    want = split(eng, out[:M])
    assert torch.equal(zh[:M], want[0]) and torch.equal(zl[:M], want[1])
    z, ez = mlp_reference(x, w1, b1, w2, b2, res)
    if norm:
        z, ez = layer_norm_reference(z, ez, lw, lb)
    check(record_property, out[:M], z, ez)


@pytest.mark.parametrize("xscale", [1e-2, 1e2])
def test_feed_forward_scaled_input(eng, record_property, xscale):
    x, w1, b1, w2, b2, res = mlp_data(300, 7, xscale)
    z, ez = mlp_reference(x, w1, b1, w2, b2, res)
    check(record_property, eng.mlp(x, w1, b1, w2, b2, res), z, ez)


def test_feed_forward_norm_with_large_common_offset(eng, record_property):
    """rows of 300 + O(0.01): the mean is removed before the variance is formed, so the normalised output keeps its accuracy
    relative to what the fp32 input rows can carry (u 300 / 0.01 ~ 2e-3 of the output's scale)"""
    M = 129
    x, w1, b1, w2, b2, _ = mlp_data(M, 11, 1e-2)
    g = torch.Generator(device=DEV).manual_seed(12)
    res = 300 + 0.01 * torch.randn(M, 256, generator=g, device=DEV)
    w2 = w2 * 0.01
    lw, lb = 1 + 0.1 * torch.randn(256, generator=g, device=DEV), 0.1 * torch.randn(256, generator=g, device=DEV)
    z, ez = mlp_reference(x, w1, b1, w2, b2, res)
    y, e = layer_norm_reference(z, ez, lw, lb)
    got = eng.mlp(x, w1, b1, w2, b2, res, ln_w=lw, ln_b=lb)
    check(record_property, got, y, e)
