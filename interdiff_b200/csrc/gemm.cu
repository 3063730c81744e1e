// GEMM front door: C[M,N] = epi(A[M,K] . W[N,K]^T)  -- nn.Linear layout, row-major, fp32 in/out.
//
// Two backends, both fp32-grade (the sampling chain is ill-conditioned, DESIGN.md "Conditioning":
// plain TF32/FP16/BF16 operand rounding diverges to O(1) over a 100-1000 step loop):
//   backend 0: fp32 SIMT register-tiled kernel (this file) -- debug / bisect path and fallback
//              for shapes the tensor-core kernel does not take.
//   backend 1: wgmma split-precision kernel on fp16 (hi, lo) operand pairs (gemm_wgmma.cu), default.
#include "common.cuh"

int idb_gemm_wgmma(idb_handle* h, const GemmArgs& g, cudaStream_t st);
bool idb_gemm_wgmma_supported(const GemmArgs& g);

namespace {

constexpr int BK = 16;

// 4 consecutive elements of an operand carried as an fp16 (hi, lo) pair: x = hi + lo * 2^-11
__device__ __forceinline__ float4 load_pair4(const __half* __restrict__ hi, const __half* __restrict__ lo, size_t off) {
    const uint2 h = *reinterpret_cast<const uint2*>(hi + off), l = *reinterpret_cast<const uint2*>(lo + off);
    const float2 h01 = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), h23 = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
    const float2 l01 = __half22float2(*reinterpret_cast<const __half2*>(&l.x)), l23 = __half22float2(*reinterpret_cast<const __half2*>(&l.y));
    const float s = 1.0f / 2048.0f;
    return make_float4(fmaf(l01.x, s, h01.x), fmaf(l01.y, s, h01.y), fmaf(l23.x, s, h23.x), fmaf(l23.y, s, h23.y));
}

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_tn_simt(const float* __restrict__ A, const __half* __restrict__ Ah, const __half* __restrict__ Al, int lda,
             const float* __restrict__ W, const __half* __restrict__ Wh, const __half* __restrict__ Wl, int ldw,
             const float* __restrict__ bias, const float* __restrict__ res, int ldr,
             float* __restrict__ C, __half* __restrict__ Cb, __half* __restrict__ Cs, int ldc, int M, int N, int K, int epi) {
    constexpr int NT = (BM / TM) * (BN / TN);
    constexpr int LA = BM * BK / 4 / NT;  // float4 loads per thread for the A tile
    constexpr int LB = BN * BK / 4 / NT;
    static_assert(LA >= 1 && LB >= 1, "tile too small for the thread count");
    __shared__ __align__(16) float As[2][BK][BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN + 4];

    const int tid = threadIdx.x;
    const int tx = tid % (BN / TN), ty = tid / (BN / TN);
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

    float4 ra[LA], rb[LB];
    auto gload = [&](int k0) {
#pragma unroll
        for (int l = 0; l < LA; l++) {
            int f = tid + l * NT, r = f / (BK / 4), kq = f % (BK / 4);
            int gm = m0 + r, gk = k0 + kq * 4;
            ra[l] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gm < M && gk < K) ra[l] = A ? *reinterpret_cast<const float4*>(A + (size_t)gm * lda + gk) : load_pair4(Ah, Al, (size_t)gm * lda + gk);
        }
#pragma unroll
        for (int l = 0; l < LB; l++) {
            int f = tid + l * NT, r = f / (BK / 4), kq = f % (BK / 4);
            int gn = n0 + r, gk = k0 + kq * 4;
            rb[l] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gn < N && gk < K) rb[l] = W ? *reinterpret_cast<const float4*>(W + (size_t)gn * ldw + gk) : load_pair4(Wh, Wl, (size_t)gn * ldw + gk);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int l = 0; l < LA; l++) {
            int f = tid + l * NT, r = f / (BK / 4), kq = f % (BK / 4);
            As[buf][kq * 4 + 0][r] = ra[l].x; As[buf][kq * 4 + 1][r] = ra[l].y;
            As[buf][kq * 4 + 2][r] = ra[l].z; As[buf][kq * 4 + 3][r] = ra[l].w;
        }
#pragma unroll
        for (int l = 0; l < LB; l++) {
            int f = tid + l * NT, r = f / (BK / 4), kq = f % (BK / 4);
            Bs[buf][kq * 4 + 0][r] = rb[l].x; Bs[buf][kq * 4 + 1][r] = rb[l].y;
            Bs[buf][kq * 4 + 2][r] = rb[l].z; Bs[buf][kq * 4 + 3][r] = rb[l].w;
        }
    };

    const int nk = (K + BK - 1) / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kb = 0; kb < nk; kb++) {
        const int buf = kb & 1;
        if (kb + 1 < nk) gload((kb + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; k++) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; i += 4) {
                float4 v = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM + i]);
                a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < TN; j += 4) {
                float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * TN + j]);
                b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
            }
#pragma unroll
            for (int i = 0; i < TM; i++)
#pragma unroll
                for (int j = 0; j < TN; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kb + 1 < nk) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }

#pragma unroll
    for (int i = 0; i < TM; i++) {
        const int gm = m0 + ty * TM + i;
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < TN; j++) {
            const int gn = n0 + tx * TN + j;
            if (gn >= N) continue;
            float v = acc[i][j];
            if (epi & EPI_BIAS) v += bias[gn];
            if (epi & EPI_GELU) v = gelu_erf(v);
            if (epi & EPI_SILU) v = silu(v);
            if (epi & EPI_RES) v += res[(size_t)gm * ldr + gn];
            if (C) C[(size_t)gm * ldc + gn] = v;
            if (Cb) split_f16(v, Cb[(size_t)gm * ldc + gn], Cs[(size_t)gm * ldc + gn]);
        }
    }
}

}  // namespace

// x[rows][cols] -> fp16 (hi, lo) pairs, zero-filling the padding columns
namespace {
__global__ void k_split_f16(const float* __restrict__ x, int ld_src, __half* __restrict__ hi, __half* __restrict__ lo, int ld_dst,
                            int rows, int cols) {
    const size_t n = (size_t)rows * ld_dst;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / ld_dst), c = (int)(i % ld_dst);
        split_f16(c < cols ? x[(size_t)r * ld_src + c] : 0.f, hi[i], lo[i]);
    }
}
}  // namespace
int idb_split_tensor(idb_handle* h, const float* x, int ld_src, __half* hi, __half* lo, int ld_dst, int rows, int cols, cudaStream_t st) {
    k_split_f16<<<296, 256, 0, st>>>(x, ld_src, hi, lo, ld_dst, rows, cols);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

int idb_gemm(idb_handle* h, const float* A, int lda, const float* W, int ldw, const float* bias,
             const float* res, int ldr, float* C, int ldc, int M, int N, int K, int epi, cudaStream_t st) {
    GemmArgs g;
    g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.bias = bias; g.res = res; g.ldr = ldr; g.C = C; g.ldc = ldc;
    g.M = M; g.N = N; g.K = K; g.epi = epi;
    return idb_gemm_ex(h, g, st);
}

int idb_gemm_ex(idb_handle* h, const GemmArgs& g_in, cudaStream_t st) {
    GemmArgs g = g_in;
    const int M = g.M, N = g.N, K = g.K;
    if (M <= 0 || N <= 0 || K <= 0) return IDB_OK;
    if ((g.C_hi == nullptr) != (g.C_lo == nullptr)) return idb_fail(h, IDB_ERR_ARG, "idb_gemm: split output needs both parts");
    if (!g.C && !g.C_hi) return idb_fail(h, IDB_ERR_ARG, "idb_gemm: no output");
    if ((!g.A && !(g.A_hi && g.A_lo)) || (!g.W && !(g.W_hi && g.W_lo))) return idb_fail(h, IDB_ERR_ARG, "idb_gemm: missing operand");
    if (h->gemm_backend == 1 && (g.ldc % 4 == 0) && (N % 4 == 0) && N >= 8) {
        // tensor-core path; fp32 operands are split into handle scratch first (stream ordered)
        const int Kp = (K + 7) & ~7;
        const size_t need = ((g.A_hi ? 0 : (size_t)M * Kp) + (g.W_hi ? 0 : (size_t)N * Kp)) * 2 * sizeof(__half) + 64;
        if (need > h->scratch_bytes) {
            if (h->scratch) { CUDA_TRY(h, cudaStreamSynchronize(st)); cudaFree(h->scratch); }
            h->scratch_bytes = need + (need >> 2);
            CUDA_TRY(h, cudaMalloc(&h->scratch, h->scratch_bytes));
        }
        __half* p = reinterpret_cast<__half*>(h->scratch);
        int rc;
        if (!g.A_hi) {
            __half* hi = p; __half* lo = p + (size_t)M * Kp; p += (size_t)2 * M * Kp;
            if ((rc = idb_split_tensor(h, g.A, g.lda, hi, lo, Kp, M, K, st))) return rc;
            g.A_hi = hi; g.A_lo = lo; g.lda = Kp;
        }
        if (!g.W_hi) {
            __half* hi = p; __half* lo = p + (size_t)N * Kp;
            if ((rc = idb_split_tensor(h, g.W, g.ldw, hi, lo, Kp, N, K, st))) return rc;
            g.W_hi = hi; g.W_lo = lo; g.ldw = Kp;
            g.pdl = 0;   // the weight pairs were produced just now on this stream: no early tile fetch
        }
        if (idb_gemm_wgmma_supported(g)) return idb_gemm_wgmma(h, g, st);
    }
    // fp32 SIMT path (prefers the full-precision operand when both forms are available); full K, plain
    // stores, so only the aux-zero side job of the tensor path has to be reproduced
    if (g.zero) CUDA_TRY(h, cudaMemset2DAsync(g.zero, sizeof(float) * g.zero_ld, 0, sizeof(float) * g.zero_cols, M, st));
    if (g_in.A) { g.A = g_in.A; g.lda = g_in.lda; }
    if (g_in.W) { g.W = g_in.W; g.ldw = g_in.ldw; }
    if ((K % 4) || (g.lda % 4) || (g.ldw % 4))
        return idb_fail(h, IDB_ERR_ARG, "idb_gemm (SIMT): K, lda, ldw must be multiples of 4 (K=%d lda=%d ldw=%d)", K, g.lda, g.ldw);
    long tiles_big = (long)((M + 127) / 128) * ((N + 63) / 64);
    if (tiles_big >= 140) {
        dim3 grid((N + 63) / 64, (M + 127) / 128);
        gemm_tn_simt<128, 64, 8, 4><<<grid, 256, 0, st>>>(g.A, g.A_hi, g.A_lo, g.lda, g.W, g.W_hi, g.W_lo, g.ldw, g.bias, g.res, g.ldr,
                                                          g.C, g.C_hi, g.C_lo, g.ldc, M, N, K, g.epi);
    } else {
        dim3 grid((N + 63) / 64, (M + 63) / 64);
        gemm_tn_simt<64, 64, 4, 4><<<grid, 256, 0, st>>>(g.A, g.A_hi, g.A_lo, g.lda, g.W, g.W_hi, g.W_lo, g.ldw, g.bias, g.res, g.ldr,
                                                         g.C, g.C_hi, g.C_lo, g.ldc, M, N, K, g.epi);
    }
    LAUNCH_CHECK(h);
    return IDB_OK;
}
