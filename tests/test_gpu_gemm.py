"""GEMM backends of the C ABI (idb_debug_gemm) against a float64 reference.  The tcgen05 backend
must be fp32-grade (split precision on fp16 (hi, lo) pairs): the bound asserted for it is the same as for the
fp32 SIMT kernel, far below plain-TF32 error (~5e-4)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from interdiff_b200.engine import Engine
    e = Engine("cuda:0")
    yield e
    e.close()


SHAPES = [(1920, 1024, 256), (1920, 256, 1024), (1920, 768, 256), (1920, 256, 256), (640, 512, 256),
          (100, 72, 36), (129, 200, 100), (1, 8, 4), (300, 1024, 260),
          (1920, 1536, 256), (2500, 1280, 200)]   # more 128-column tiles than the H100 has SMs (132): several waves


@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_matches_fp64(eng, backend, shape):
    M, N, K = shape
    eng.set_gemm_backend(backend)
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    ref = A.double() @ W.double().T
    out = eng.gemm(A, W).cpu().double()
    scale = ref.abs().max()
    assert ((out - ref).abs().max() / scale).item() < 2e-6
    out = eng.gemm(A, W, bias=bias, res=res, gelu=True).cpu().double()
    ref2 = torch.nn.functional.gelu(ref + bias.double()) + res.double()
    assert ((out - ref2).abs().max() / ref2.abs().max()).item() < 2e-6
    eng.set_gemm_backend("simt")


def test_tcgen05_beats_plain_tf32_precision(eng):
    """Property: the split-precision kernel is >= 100x more accurate than single-pass TF32 would be."""
    eng.set_gemm_backend("tcgen05")
    g = torch.Generator().manual_seed(5)
    A = torch.randn(512, 1024, generator=g)
    W = torch.randn(256, 1024, generator=g)
    ref = A.double() @ W.double().T
    err = ((eng.gemm(A, W).cpu().double() - ref).abs().max() / ref.abs().max()).item()
    tf32 = lambda x: (x.view(torch.int32) + 0x1000 & ~0x1FFF).view(torch.float32)
    err_tf32 = ((tf32(A.clone()).double() @ tf32(W.clone()).double().T - ref).abs().max() / ref.abs().max()).item()
    eng.set_gemm_backend("simt")
    assert err < err_tf32 / 100, (err, err_tf32)


@pytest.mark.parametrize("shape", [(1920, 256, 1024), (300, 64, 260), (129, 200, 128), (64, 8, 64)])
def test_split_k_matches_fp64_and_is_deterministic(eng, shape):
    """2-way split-K (how the denoiser runs ff2): partial tiles are reduced with fp32 atomics onto a
    zeroed C; with two addends the order cannot matter, so repeated runs must agree bit for bit."""
    M, N, K = shape
    eng.set_gemm_backend("tcgen05")
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    ref = A.double() @ W.double().T + bias.double() + res.double()
    outs = [eng.gemm(A, W, bias=bias, res=res, split_k=True).cpu() for _ in range(3)]
    eng.set_gemm_backend("simt")
    assert ((outs[0].double() - ref).abs().max() / ref.abs().max()).item() < 2e-6
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
def test_gelu_epilogue_accuracy_on_a_grid(eng, backend):
    """The epilogue's erf-GELU (branch-free minimax fit, common.cuh) against float64 on every multiple of
    2^-10 in [-8, 8]: the inputs are exactly representable by the fp16 (hi, lo) operand pairs and the
    'GEMM' is a multiplication by the identity, so the only error left is the activation's."""
    eng.set_gemm_backend(backend)
    x = (torch.arange(-8 * 1024, 8 * 1024 + 1, dtype=torch.float32) / 1024.0)
    x = x[: (x.numel() // 8) * 8].reshape(-1, 8)
    out = eng.gemm(x, torch.eye(8), gelu=True).cpu().double()
    eng.set_gemm_backend("simt")
    ref = torch.nn.functional.gelu(x.double())
    # erf error <= 1.0e-7 (fit) -> GELU error <= 0.5 |x| 1e-7, plus the fp32 rounding of the result
    bound = 2.5e-7 * torch.clamp(x.double().abs(), min=1.0)
    assert bool(((out - ref).abs() <= bound).all()), ((out - ref).abs() / bound).max().item()


@pytest.mark.parametrize("M", [1920, 129, 5])
def test_fused_feed_forward_kernel(eng, M):
    """The cluster kernel gelu(x W1^T + b1) W2^T + b2 + res (8 CTAs exchange partial tiles over distributed
    shared memory) against float64; the rank-ordered reduction makes it bit-reproducible."""
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, 256, generator=g)
    w1 = torch.randn(1024, 256, generator=g) / 16
    b1 = torch.randn(1024, generator=g) * 0.1
    w2 = torch.randn(256, 1024, generator=g) / 32
    b2 = torch.randn(256, generator=g) * 0.1
    res = torch.randn(M, 256, generator=g)
    ref = torch.nn.functional.gelu(x.double() @ w1.double().T + b1.double()) @ w2.double().T + b2.double() + res.double()
    outs = [eng.mlp(x, w1, b1, w2, b2, res).cpu() for _ in range(3)]
    assert ((outs[0].double() - ref).abs().max() / ref.abs().max()).item() < 2e-6
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
