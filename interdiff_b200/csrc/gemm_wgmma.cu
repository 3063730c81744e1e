// wgmma split-precision GEMM for sm_90a:  C[M,N] = epi(A[M,K] . W[N,K]^T), fp32-grade accuracy.
//
// Why split precision: the sampling chain amplifies operand rounding (DESIGN.md "Conditioning"),
// so the tensor-core path has to be fp32-grade.  Every fp32 operand x is carried as a pair of fp16
//     hi = fp16_rn(x),   lo = fp16_rn((x - hi) * 2^11)          (x - hi is exact in fp32)
// so that x = hi + lo * 2^-11 up to max(2^-23 |x|, 2^-36), and
//     A W^T = A_hi W_hi^T  +  2^-11 (A_lo W_hi^T + A_hi W_lo^T)  (+ 2^-22 A_lo W_lo^T, dropped).
// The 2^11 scale keeps `lo` a normal fp16 number while |x - hi| >= 2^-25; below that lo is subnormal (spacing 2^-24, i.e.
// 2^-35 in units of x), so the relative 2^-23 holds for |x| >= 2^-13 and smaller operands carry an absolute error of at
// most 2^-36 (for |x| < 2^-14 hi itself is subnormal).  tests/test_gpu_gemm_kernels.py checks this floor element by element.
// The two sums accumulate in SEPARATE fp32 register accumulators and are combined in the epilogue.
// Range: |x| < 65504 (activations and weights of this model are O(1e-3 .. 1e3)).
//
// Pipeline per CTA (128 x BN output tiles, 288 threads; the 64-column kernel is persistent, see gemm_split_f16_persistent):
//   warp 8    : TMA producer (warp-uniform loop, one elected lane issues): 4 x cp.async.bulk.tensor.2d per
//               stage (A_hi, W_hi, A_lo, W_lo k-blocks of 64 fp16 = one 128B-swizzle row), mbarrier tx.
//   warps 0-7 : two consumer warpgroups, 64 rows of the tile each: 12 wgmma.mma_async m64nBNk16 per k-block
//               (4 k-steps of 16 x {lo*hi, hi*lo -> small; hi*hi -> main}), release of the stage, then the
//               epilogue: sum, bias / GELU / SiLU, residual, stores (128-column kernels: straight from the accumulator
//               registers, a quad of lanes covers one 32-byte sector of a row; 64-column kernel: staged through shared
//               memory, whole rows); optional output already split into (hi, lo) fp16 pairs for the next GEMM.
// The tensor core truncates on every fp32 accumulate, so the hi*hi products of every k-block (or of `promote`
// k-blocks) go into a fresh accumulator that is then added to the running sum with an IEEE fp32 addition.  The order
// of the additions per output element is a function of K alone - not of the tile width or of M.
#include "common.cuh"
#include "tc_mlp.cuh"

#include <cuda.h>

namespace {

using namespace tc;

constexpr int GEMM_CW = 8;                           // consumer warps (two warpgroups)
constexpr int GEMM_THREADS = (GEMM_CW + 1) * 32;     // + TMA producer

template <int BN> struct Cfg {
    static constexpr int A_BYTES = BM * BK * 2;               // 16 KB
    static constexpr int W_BYTES = BN * BK * 2;
    static constexpr int HALF_BYTES = A_BYTES + W_BYTES;      // [A_hi | W_hi], then the same for lo
    static constexpr int STAGE_BYTES = 2 * HALF_BYTES;
    static constexpr int STAGES = (BN == 128) ? 3 : 4;       // 192 KB of the SM's 227 KB either way
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

// MC (multicast pairs): launched with cluster dimensions (1, 2, 1) - the two CTAs of a cluster own two ROW tiles of the same
// column tile.  Each loads its own A tile and HALF of the shared W tile, multicast into both CTAs' shared memory
// (cp.async.bulk.tensor ... .multicast::cluster), which halves the L2 -> SM traffic of the W operand; a stage is refilled only
// when the consumers of BOTH CTAs have released it (each consumer warp arrives on the "empty" barrier of both).
template <int BN, bool MC = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_split_f16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                      const __grid_constant__ CUtensorMap map_al, const __grid_constant__ CUtensorMap map_wl,
                      const float* __restrict__ bias, const float* __restrict__ res, int ldr,
                      float* __restrict__ C, __half* __restrict__ Ch, __half* __restrict__ Cl, int ldc, int M, int N, int K, int epi,
                      int promote, float* __restrict__ zero_ptr, int zero_ld, int zero_cols, long long* __restrict__ trace) {
    using cfg = Cfg<BN>;
    constexpr int NR = BN / 2;               // accumulator registers per thread
    // optional per-CTA timeline (clock64 at named points) for debugging the pipeline
    long long* tr = trace ? trace + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 16 : nullptr;
#define TRACE(slot) do { if (tr) tr[slot] = clock64(); } while (0)
    if (threadIdx.x == 0) { TRACE(0); chain_mark(1, 0); }
    pdl_trigger();   // the next kernel may start its own prologue now (it blocks in pdl_wait before touching our output)
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bars = base + cfg::STAGES * cfg::STAGE_BYTES;
    // barrier layout (8 B each): full[S], empty[S]
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (cfg::STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    // split-K: blockIdx.z owns a contiguous range of k-blocks; the partial tiles are combined with
    // fp32 reductions onto a zeroed C (two addends only, so the result does not depend on their order)
    const int total_kb = (K + BK - 1) / BK, per_kb = (total_kb + gridDim.z - 1) / gridDim.z;
    const int kb0 = blockIdx.z * per_kb;
    const int num_kb = min(per_kb, total_kb - kb0);

    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg::STAGES; s++) {
            mbar_init(bar_full(s), 1);
            mbar_init(bar_empty(s), MC ? 2 * GEMM_CW : GEMM_CW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_al) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_wl) : "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) TRACE(1);
    uint32_t crank = 0;
    if (MC) {
        asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(crank));
        cluster_sync_all();      // the peer's barriers exist before anything is multicast into its shared memory
    }
    constexpr int WH = cfg::W_BYTES / 2;     // bytes of half a W tile (MC: the part this CTA fetches for both)

    if (warp == GEMM_CW) {
        // ===================== TMA producer =====================
        // The weight tiles of the first pipeline fill do not depend on the previous kernel: requested before the dependency
        // wait, the activation tiles after.
        const int npre = num_kb < cfg::STAGES ? num_kb : cfg::STAGES;
        auto load_w = [&](int s, int kb) {
            const uint32_t dst = base + s * cfg::STAGE_BYTES;
            if (MC) {
                tma_load_2d_mc(dst + cfg::A_BYTES + crank * WH, &map_w, bar_full(s), (kb0 + kb) * BK, n0 + crank * (BN / 2), 3);
                tma_load_2d_mc(dst + cfg::HALF_BYTES + cfg::A_BYTES + crank * WH, &map_wl, bar_full(s), (kb0 + kb) * BK, n0 + crank * (BN / 2), 3);
            } else {
                tma_load_2d(dst + cfg::A_BYTES, &map_w, bar_full(s), (kb0 + kb) * BK, n0);
                tma_load_2d(dst + cfg::HALF_BYTES + cfg::A_BYTES, &map_wl, bar_full(s), (kb0 + kb) * BK, n0);
            }
        };
        auto load_a = [&](int s, int kb) {
            const uint32_t dst = base + s * cfg::STAGE_BYTES;
            tma_load_2d(dst, &map_a, bar_full(s), (kb0 + kb) * BK, m0);
            tma_load_2d(dst + cfg::HALF_BYTES, &map_al, bar_full(s), (kb0 + kb) * BK, m0);
        };
        if (elect_one()) {
            for (int kb = 0; kb < npre; kb++) { mbar_arrive_expect_tx(bar_full(kb), cfg::STAGE_BYTES); load_w(kb, kb); }
        }
        __syncwarp();
        pdl_wait();
        if (lane == 0) chain_mark(1, 1);
        if (elect_one()) {
            for (int kb = 0; kb < npre; kb++) load_a(kb, kb);
        }
        __syncwarp();
        if (lane == 0) TRACE(2);
        for (int kb = npre; kb < num_kb; kb++) {
            const int s = kb % cfg::STAGES, round = kb / cfg::STAGES;
            mbar_wait(bar_empty(s), (round - 1) & 1);
            if (elect_one()) {
                mbar_arrive_expect_tx(bar_full(s), cfg::STAGE_BYTES);
                load_a(s, kb);
                load_w(s, kb);
            }
            __syncwarp();
        }
        if (lane == 0) TRACE(3);
    } else {
        // ===================== consumer warpgroups =====================
        const int wg = warp >> 2;
        const uint32_t a_off = (uint32_t)wg * 8192u;     // the warpgroup's 64 rows of the A tile
        pdl_wait();      // bias / residual reads and the stores below touch buffers of earlier kernels
        if (zero_ptr) {
            // side job: clear this CTA's patch of an auxiliary matrix (the zeroed C that the NEXT split-K GEMM reduces into)
            const int zc4 = zero_cols / (int)gridDim.x / 4;
            for (int i = threadIdx.x; i < BM * zc4; i += GEMM_CW * 32) {
                const int r = i / zc4, c4 = i % zc4;
                if (m0 + r < M)
                    *reinterpret_cast<float4*>(zero_ptr + (size_t)(m0 + r) * zero_ld + (blockIdx.x * zc4 + c4) * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        float sum[NR], part[NR], small[NR];
#pragma unroll
        for (int i = 0; i < NR; i++) sum[i] = 0.f;
        for (int kb = 0; kb < num_kb; kb++) {
            const int s = kb % cfg::STAGES, round = kb / cfg::STAGES;
            mbar_wait(bar_full(s), round & 1);
            if (kb == 0 && threadIdx.x == 0) TRACE(6);
            const uint32_t a_hi = base + s * cfg::STAGE_BYTES + a_off, w_hi = base + s * cfg::STAGE_BYTES + cfg::A_BYTES;
            wgmma_fence();
            // debug bit 64: hi x hi only (MMA throughput probe)
            split_kblock(part, small, make_smem_desc(a_hi), make_smem_desc(a_hi + cfg::HALF_BYTES), make_smem_desc(w_hi),
                         make_smem_desc(w_hi + cfg::HALF_BYTES), kb % promote == 0, kb == 0, !(epi & 64));
            wgmma_commit();
            wgmma_wait0();
            __syncwarp();
            if (lane == 0) {       // stage reusable once this warp's MMAs have read it
                mbar_arrive(bar_empty(s));
                if (MC) mbar_arrive_remote(bar_empty(s), crank ^ 1u);      // ... in BOTH CTAs of the pair (each multicasts into the other's stage)
            }
            if ((kb + 1) % promote == 0 || kb == num_kb - 1) {
#pragma unroll
                for (int i = 0; i < NR; i++) sum[i] += part[i];
            }
        }
        if (threadIdx.x == 0) TRACE(9);
        // ---- epilogue from the accumulator layout: thread = rows r0, r0 + 8; columns 8 j + cq, + 1
        const bool splitk = gridDim.z > 1, lead = blockIdx.z == 0;
        const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
            const int col = n0 + 8 * j + cq;      // even, and N is a multiple of 4: col < N implies col + 1 < N
            if (col >= N) continue;
            float2 b2 = make_float2(0.f, 0.f);
            if ((epi & EPI_BIAS) && lead) b2 = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                const int row = r0 + 8 * hh;
                if (row >= M) continue;
                float2 o;
                if (epi & 64) o = make_float2(sum[4 * j + 2 * hh], sum[4 * j + 2 * hh + 1]);
                else o = make_float2(fmaf(small[4 * j + 2 * hh], 1.0f / 2048.0f, sum[4 * j + 2 * hh]),
                                     fmaf(small[4 * j + 2 * hh + 1], 1.0f / 2048.0f, sum[4 * j + 2 * hh + 1]));
                o.x += b2.x; o.y += b2.y;
                if (epi & EPI_GELU) { o.x = gelu_erf(o.x); o.y = gelu_erf(o.y); }
                if (epi & EPI_SILU) { o.x = silu(o.x); o.y = silu(o.y); }
                if ((epi & EPI_RES) && lead) {
                    const float2 r2 = *reinterpret_cast<const float2*>(res + (size_t)row * ldr + col);
                    o.x += r2.x; o.y += r2.y;
                }
                if (splitk) {
                    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(C + (size_t)row * ldc + col), "f"(o.x), "f"(o.y) : "memory");
                } else if (C) *reinterpret_cast<float2*>(C + (size_t)row * ldc + col) = o;
                if (Ch) {
                    __half2 h01, l01;
                    split_f16x2(o.x, o.y, h01, l01);
                    *reinterpret_cast<__half2*>(Ch + (size_t)row * ldc + col) = h01;
                    *reinterpret_cast<__half2*>(Cl + (size_t)row * ldc + col) = l01;
                }
            }
        }
        if (threadIdx.x == 0) TRACE(10);
    }
    __syncthreads();
    if (MC) cluster_sync_all();      // the peer may still arrive on this CTA's barriers until it is done too
    if (threadIdx.x == 0) { TRACE(11); chain_mark(1, 2); }
#undef TRACE
}

// Persistent 64-column kernel (every GEMM that does not take the 128-column kernels above).  Grid (cpr, gy, ksplit), at most
// one CTA per SM: CTA (x, y) owns the contiguous run of column tiles [x ct / cpr, (x + 1) ct / cpr) of row tiles y, y + gy, ..
// (ct = column tiles).  The schedule is a function of the shape and the SM count only, and an element's additions are the
// same whatever CTA computes its tile.
// Shared memory: A ring of 4 slots of 32 KB (a k-block of the 128-row tile: hi 16 KB | lo 16 KB), W ring of 4 slots of 16 KB
// (hi 8 KB | lo 8 KB), each with full / empty barriers.  When the CTA's k-blocks fit into the A ring (K <= 256 per split), a
// row tile's A block is loaded once and stays resident across the CTA's column tiles, released after the last of them: A
// traffic drops by the column tiles per CTA.  Otherwise A streams with W, one A slot per k-block.  The producer runs ahead
// across tile boundaries, so the next tile's loads are in flight while the consumers run the epilogue.
namespace pers {
constexpr int A_SLOTS = 4, W_SLOTS = 4;
constexpr int A_BYTES = 2 * BM * BK * 2;       // hi | lo
constexpr int W_BYTES = 2 * 64 * BK * 2;       // hi | lo
constexpr int W_OFF = A_SLOTS * A_BYTES;
constexpr int E_OFF = W_OFF + W_SLOTS * W_BYTES;
constexpr int E_BYTES = 16 * 64 * 4;           // a consumer warp's 16 x 64 fp32 rows of the tile, staged for the epilogue
constexpr int SMEM_BYTES = E_OFF + GEMM_CW * E_BYTES + 1024 /*align*/ + 256 /*barriers*/;     // 224 KB + 1.25 KB
}  // namespace pers

__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_split_f16_persistent(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                          const __grid_constant__ CUtensorMap map_al, const __grid_constant__ CUtensorMap map_wl,
                          const float* __restrict__ bias, const float* __restrict__ res, int ldr,
                          float* __restrict__ C, __half* __restrict__ Ch, __half* __restrict__ Cl, int ldc, int M, int N, int K, int epi,
                          int promote, float* __restrict__ zero_ptr, int zero_ld, int zero_cols, long long* __restrict__ trace) {
    using namespace pers;
    constexpr int BN = 64, NR = BN / 2;
    const long long t_entry = clock64();
    if (threadIdx.x == 0) chain_mark(1, 0);
    pdl_trigger();   // the next kernel may start its own prologue now (it blocks in pdl_wait before touching our output)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bars = base + E_OFF + GEMM_CW * E_BYTES;
    // barriers (8 B each): a_full[4], a_empty[4], w_full[4], w_empty[4]
    auto a_full = [&](int s) { return bars + 8u * s; };
    auto a_empty = [&](int s) { return bars + 8u * (A_SLOTS + s); };
    auto w_full = [&](int s) { return bars + 8u * (2 * A_SLOTS + s); };
    auto w_empty = [&](int s) { return bars + 8u * (2 * A_SLOTS + W_SLOTS + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ct = (N + BN - 1) / BN, rt = (M + BM - 1) / BM;
    const int c_begin = blockIdx.x * ct / gridDim.x, ncols = (blockIdx.x + 1) * ct / gridDim.x - c_begin;
    const int nrows = (rt - blockIdx.y + gridDim.y - 1) / gridDim.y;
    // split-K: blockIdx.z owns a contiguous range of k-blocks; the partial tiles are combined with
    // fp32 reductions onto a zeroed C (two addends only, so the result does not depend on their order)
    const int total_kb = (K + BK - 1) / BK, per_kb = (total_kb + gridDim.z - 1) / gridDim.z;
    const int kb0 = blockIdx.z * per_kb;
    const int num_kb = min(per_kb, total_kb - kb0);
    const bool resident = num_kb <= A_SLOTS;
    const int total_w = nrows * ncols * num_kb;      // W k-blocks this CTA loads, in consumption order
    // item i (one k-block of one tile) -> row tile, column tile
    auto item_row = [&](int i) { return blockIdx.y + (i / num_kb / ncols) * gridDim.y; };
    auto item_col = [&](int i) { return c_begin + (i / num_kb) % ncols; };
    // optional per-tile timeline (clock64 at named points; profiles/gemm_trace.py lists the slots), one record per tile
    auto rec = [&](int r, int c) { return trace ? trace + ((size_t)r * ct + c) * 16 : nullptr; };
    long long* const tr_first = rec(blockIdx.y, c_begin);

    if (threadIdx.x == 0) {
        for (int s = 0; s < A_SLOTS; s++) { mbar_init(a_full(s), 1); mbar_init(a_empty(s), GEMM_CW); }
        for (int s = 0; s < W_SLOTS; s++) { mbar_init(w_full(s), 1); mbar_init(w_empty(s), GEMM_CW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_al) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_wl) : "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0 && tr_first) { tr_first[0] = t_entry; tr_first[1] = clock64(); }

    if (warp == GEMM_CW) {
        // ===================== TMA producer =====================
        auto load_w = [&](int i) {
            const int s = i % W_SLOTS;
            const uint32_t dst = base + W_OFF + s * W_BYTES;
            const int k = (kb0 + i % num_kb) * BK, n0 = item_col(i) * BN;
            mbar_arrive_expect_tx(w_full(s), W_BYTES);
            tma_load_2d(dst, &map_w, w_full(s), k, n0);
            tma_load_2d(dst + W_BYTES / 2, &map_wl, w_full(s), k, n0);
        };
        // The first W k-blocks do not depend on the previous kernel: requested before the dependency wait.
        const int npre = min(total_w, W_SLOTS);
        if (elect_one()) {
            for (int i = 0; i < npre; i++) load_w(i);
        }
        __syncwarp();
        pdl_wait();
        if (lane == 0) chain_mark(1, 1);
        int ai = 0;      // A k-blocks loaded so far
        for (int i = 0; i < total_w; i++) {
            if (!resident || item_col(i) == c_begin) {
                const int s = ai % A_SLOTS;
                if (ai >= A_SLOTS) mbar_wait(a_empty(s), (ai / A_SLOTS - 1) & 1);
                if (elect_one()) {
                    const uint32_t dst = base + s * A_BYTES;
                    const int k = (kb0 + i % num_kb) * BK, m0 = item_row(i) * BM;
                    mbar_arrive_expect_tx(a_full(s), A_BYTES);
                    tma_load_2d(dst, &map_a, a_full(s), k, m0);
                    tma_load_2d(dst + A_BYTES / 2, &map_al, a_full(s), k, m0);
                }
                __syncwarp();
                ai++;
            }
            if (i >= npre) {
                mbar_wait(w_empty(i % W_SLOTS), (i / W_SLOTS - 1) & 1);
                if (elect_one()) load_w(i);
                __syncwarp();
            }
            if (i == 0 && lane == 0 && tr_first) tr_first[2] = clock64();
        }
        if (lane == 0 && tr_first) tr_first[3] = clock64();
    } else {
        // ===================== consumer warpgroups =====================
        const int wg = warp >> 2;
        const uint32_t a_off = (uint32_t)wg * 8192u;     // the warpgroup's 64 rows of the A tile
        pdl_wait();      // bias / residual reads and the stores below touch buffers of earlier kernels
        const bool splitk = gridDim.z > 1, lead = blockIdx.z == 0;
        int i = 0, ag = 0;     // W k-blocks consumed; A k-blocks of the tiles before the current A group
        for (int rr = 0; rr < nrows; rr++) {
            const int r = blockIdx.y + rr * gridDim.y, m0 = r * BM;
            for (int cc = 0; cc < ncols; cc++) {
                const int c = c_begin + cc, n0 = c * BN;
                long long* const tr = rec(r, c);
                if (threadIdx.x == 0 && tr && (rr || cc)) tr[0] = clock64();
                const bool last_use = !resident || cc == ncols - 1;      // of the A k-blocks
                if (zero_ptr) {
                    // side job: clear this tile's patch of an auxiliary matrix (the zeroed C that the NEXT split-K GEMM reduces into)
                    const int zc4 = zero_cols / ct / 4;
                    for (int j = threadIdx.x; j < BM * zc4; j += GEMM_CW * 32) {
                        const int rz = j / zc4, c4 = j % zc4;
                        if (m0 + rz < M)
                            *reinterpret_cast<float4*>(zero_ptr + (size_t)(m0 + rz) * zero_ld + (c * zc4 + c4) * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
                float sum[NR], part[NR], small[NR];
#pragma unroll
                for (int j = 0; j < NR; j++) sum[j] = 0.f;
                for (int kb = 0; kb < num_kb; kb++, i++) {
                    const int sa = (ag + kb) % A_SLOTS, sw = i % W_SLOTS;
                    mbar_wait(a_full(sa), ((ag + kb) / A_SLOTS) & 1);
                    mbar_wait(w_full(sw), (i / W_SLOTS) & 1);
                    if (kb == 0 && threadIdx.x == 0 && tr) tr[6] = clock64();
                    const uint32_t a_hi = base + sa * A_BYTES + a_off, w_hi = base + W_OFF + sw * W_BYTES;
                    wgmma_fence();
                    // debug bit 64: hi x hi only (MMA throughput probe)
                    split_kblock(part, small, make_smem_desc(a_hi), make_smem_desc(a_hi + A_BYTES / 2), make_smem_desc(w_hi),
                                 make_smem_desc(w_hi + W_BYTES / 2), kb % promote == 0, kb == 0, !(epi & 64));
                    wgmma_commit();
                    wgmma_wait0();
                    __syncwarp();
                    if (lane == 0) {       // slots reusable once this warp's MMAs have read them
                        mbar_arrive(w_empty(sw));
                        if (last_use) mbar_arrive(a_empty(sa));
                    }
                    if ((kb + 1) % promote == 0 || kb == num_kb - 1) {
#pragma unroll
                        for (int j = 0; j < NR; j++) sum[j] += part[j];
                    }
                }
                if (last_use) ag += num_kb;
                if (threadIdx.x == 0 && tr) tr[9] = clock64();
                // ---- epilogue.  The warp's 16 rows of sum + 2^-11 small go through shared memory (accumulator layout in: rows
                // lane / 4 (+ 8), columns 8 j + 2 (lane % 4); XOR swizzle of the column by 8 (row % 4) keeps the float2 writes of a
                // half-warp on distinct banks), then out row by row, 16 lanes x float4 per row: every store instruction writes two
                // whole 256-byte row segments instead of 8-byte pieces of 8 rows.  Then bias / GELU / SiLU, residual, stores.
                float* const stage = reinterpret_cast<float*>(smem_raw + (base - smem_u32(smem_raw)) + E_OFF + warp * E_BYTES);
                {
                    const int rl = lane >> 2, cq = 2 * (lane & 3);
#pragma unroll
                    for (int j = 0; j < BN / 8; j++) {
#pragma unroll
                        for (int hh = 0; hh < 2; hh++) {
                            const int row = rl + 8 * hh, e = 4 * j + 2 * hh;
                            const float2 v = (epi & 64) ? make_float2(sum[e], sum[e + 1])
                                                        : make_float2(fmaf(small[e], 1.0f / 2048.0f, sum[e]), fmaf(small[e + 1], 1.0f / 2048.0f, sum[e + 1]));
                            *reinterpret_cast<float2*>(stage + row * BN + ((8 * j + cq) ^ (8 * (row & 3)))) = v;
                        }
                    }
                }
                __syncwarp();
                {
                    const int cl = 4 * (lane & 15), col = n0 + cl;      // N is a multiple of 4: col < N implies col + 3 < N
                    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
                    if ((epi & EPI_BIAS) && lead && col < N) b4 = *reinterpret_cast<const float4*>(bias + col);
#pragma unroll 2
                    for (int it = 0; it < 8; it++) {
                        const int rl = 2 * it + (lane >> 4), row = m0 + wg * 64 + (warp & 3) * 16 + rl;
                        if (row >= M || col >= N) continue;
                        float4 o = *reinterpret_cast<const float4*>(stage + rl * BN + (cl ^ (8 * (rl & 3))));
                        o.x += b4.x; o.y += b4.y; o.z += b4.z; o.w += b4.w;
                        if (epi & EPI_GELU) { o.x = gelu_erf(o.x); o.y = gelu_erf(o.y); o.z = gelu_erf(o.z); o.w = gelu_erf(o.w); }
                        if (epi & EPI_SILU) { o.x = silu(o.x); o.y = silu(o.y); o.z = silu(o.z); o.w = silu(o.w); }
                        if ((epi & EPI_RES) && lead) {
                            const float4 r4 = *reinterpret_cast<const float4*>(res + (size_t)row * ldr + col);
                            o.x += r4.x; o.y += r4.y; o.z += r4.z; o.w += r4.w;
                        }
                        if (splitk) {
                            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(C + (size_t)row * ldc + col), "f"(o.x), "f"(o.y),
                                         "f"(o.z), "f"(o.w) : "memory");
                        } else if (C) *reinterpret_cast<float4*>(C + (size_t)row * ldc + col) = o;
                        if (Ch) {
                            __half2 h01, l01, h23, l23;
                            split_f16x2(o.x, o.y, h01, l01);
                            split_f16x2(o.z, o.w, h23, l23);
                            *reinterpret_cast<uint2*>(Ch + (size_t)row * ldc + col) = make_uint2(*reinterpret_cast<uint32_t*>(&h01), *reinterpret_cast<uint32_t*>(&h23));
                            *reinterpret_cast<uint2*>(Cl + (size_t)row * ldc + col) = make_uint2(*reinterpret_cast<uint32_t*>(&l01), *reinterpret_cast<uint32_t*>(&l23));
                        }
                    }
                }
                __syncwarp();      // the staging rows are rewritten by the next tile
                if (threadIdx.x == 0 && tr) tr[10] = clock64();
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long* const tr = rec(blockIdx.y + (nrows - 1) * gridDim.y, c_begin + ncols - 1);
        if (tr) { tr[11] = clock64(); if (tr != tr_first) tr[12] = t_entry; }
        chain_mark(1, 2);
    }
}

// stand-alone launch of the feed-forward block: grid (8, ceil(M / 128)), one 128-row tile per cluster
__global__ void __cluster_dims__(mlp::CLUSTER, 1, 1) __launch_bounds__(NUM_THREADS, 1)
mlp_fused_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w1,
                 const __grid_constant__ CUtensorMap map_xl, const __grid_constant__ CUtensorMap map_w1l,
                 const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_w2l,
                 const float* __restrict__ b1, const float* __restrict__ b2, const float* __restrict__ res, int ldr,
                 float* __restrict__ Z, int ldz, int M, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                 __half* __restrict__ Zh, __half* __restrict__ Zl, long long* __restrict__ trace) {
    long long* tr = trace ? trace + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 16 : nullptr;
    if (tr && threadIdx.x == 0) tr[0] = clock64();
    if (threadIdx.x == 0) chain_mark(2, 0);
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    MlpArgs a{&map_x, &map_w1, &map_xl, &map_w1l, &map_w2, &map_w2l, b1, b2, res, ldr, Z, ldz, ln_w, ln_b, Zh, Zl};
    mlp_tile(smem_raw, a, blockIdx.x, blockIdx.y * BM, M, tr);
    if (threadIdx.x == 0) chain_mark(2, 2);
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int make_map(idb_handle* h, CUtensorMap* map, const __half* ptr, int rows, int cols, int ld, int box_rows) {
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        CUDA_TRY(h, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        if (!fn || qres != cudaDriverEntryPointSuccess) return idb_fail(h, IDB_ERR_CUDA, "cuTensorMapEncodeTiled not available");
        g_encode = (EncodeTiledFn)fn;
    }
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)ptr, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return idb_fail(h, IDB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return IDB_OK;
}

}  // namespace

CHAIN_SETTER(idb_chain_set_gemm)
long long* g_idb_gemm_trace = nullptr;   // set by the debug hooks for ONE following launch
int g_idb_gemm_wide_tiles = 1;           // 128-column tiles where idb_gemm_wgmma picks them; 0 = 64-column tiles everywhere (test hook)
int g_idb_gemm_promote = 0;              // 0 = default; test hook (idb_debug_set_gemm_accumulators)
int g_idb_gemm_persistent = 1;           // 0 = one tile per CTA in the 64-column kernel (test hook)

bool idb_gemm_wgmma_supported(const GemmArgs& g) {
    // TMA needs 16-byte aligned row strides (8 fp16); the vector epilogue needs ldc % 4 == 0
    return g.A_lo && g.W_lo && g.M >= 1 && g.N >= 8 && g.K >= 8 && (g.lda % 8 == 0) && (g.ldw % 8 == 0) && (g.ldc % 4 == 0) &&
           (g.N % 4 == 0);
}

int idb_gemm_wgmma(idb_handle* h, const GemmArgs& g, cudaStream_t st) {
    long long* trace = g_idb_gemm_trace;
    g_idb_gemm_trace = nullptr;
    const int M = g.M, N = g.N, K = g.K;
    auto mis = [](const void* p) { return ((uintptr_t)p & 15) != 0; };
    if (mis(g.A_hi) || mis(g.W_hi) || mis(g.A_lo) || mis(g.W_lo) || mis(g.C) || mis(g.C_hi) || mis(g.C_lo))
        return idb_fail(h, IDB_ERR_ARG, "wgmma GEMM needs 16-byte aligned pointers");
    if ((g.epi & EPI_RES) && ((g.ldr % 4) || mis(g.res))) return idb_fail(h, IDB_ERR_ARG, "residual must be 16-byte aligned");
    if ((g.epi & EPI_BIAS) && mis(g.bias)) return idb_fail(h, IDB_ERR_ARG, "bias must be 16-byte aligned");
    if (!(h->attr_mask & 1u)) {      // per handle = per device (function attributes live in the device's context)
        CUDA_TRY(h, cudaFuncSetAttribute(gemm_split_f16_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<128>::SMEM_BYTES));
        CUDA_TRY(h, cudaFuncSetAttribute(gemm_split_f16_persistent, cudaFuncAttributeMaxDynamicSharedMemorySize, pers::SMEM_BYTES));
        CUDA_TRY(h, cudaFuncSetAttribute(gemm_split_f16_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<128>::SMEM_BYTES));
        h->attr_mask |= 1u;
    }
    // wide single-accumulator outputs take 128-column tiles; everything else 64, so more SMs get a tile.  With the per-k-block
    // fp32 promotion the 128-column kernel holds three 64-float accumulator sets at its 168-register cap and spills inside
    // the k-loop: on an H100 it ran the 1920 x 1536 x 256 attention-projection GEMM in 37 us against 29 us for 64-column
    // tiles.  A tile's width does not change any element's result (same operations in the same order), so the choice is free.
    const int row_tiles = (M + BM - 1) / BM;
    const long tiles128 = (long)row_tiles * ((N + 127) / 128);
    const bool wide = g_idb_gemm_wide_tiles && g.single_acc && 2 * tiles128 >= h->sm_count;
    CUtensorMap ma, mw, mal, mwl;
    int rc;
    if ((rc = make_map(h, &ma, g.A_hi, M, K, g.lda, BM))) return rc;
    if ((rc = make_map(h, &mal, g.A_lo, M, K, g.lda, BM))) return rc;
    // split-K (2 only: two addends commute, so the reduction order cannot change the result) needs a C that
    // an earlier kernel zeroed (GemmArgs::zero of the producer GEMM) and the plain fp32 output
    int ksplit = g.ksplit == 2 && (K + BK - 1) / BK >= 2 ? 2 : 1;
    if (ksplit == 2 && (!g.C || g.C_hi || (g.epi & (EPI_GELU | EPI_SILU))))
        return idb_fail(h, IDB_ERR_ARG, "split-K GEMM: fp32 output only, no activation");
    float* zero = g.zero;
    if (zero) {
        const int gx = wide ? (N + 127) / 128 : (N + 63) / 64;
        if (g.zero_cols % (4 * gx) || (g.zero_ld & 3)) return idb_fail(h, IDB_ERR_ARG, "aux zero: %d columns do not split over %d column tiles", g.zero_cols, gx);
    }
    // k-blocks accumulated inside the tensor core between two fp32 promotions: 1 bounds the truncate-on-accumulate error at
    // 4 k-steps whatever K is; a caller for whom one tensor-core accumulator is accurate enough (single_acc, e.g. the mm-scale
    // pose blend added to metre-scale vertices) skips the promotions.  A function of the call, never of M, so that a sample's
    // result does not depend on how many samples share the batch (multi-GPU runs slice one global batch; SURVEY 8e).
    int promote = g.single_acc ? (1 << 30) : 1;
    if (g_idb_gemm_promote > 0) promote = g_idb_gemm_promote;
    if (wide && h->gemm_multicast && row_tiles >= 2 && ksplit == 1 && !zero) {
        // long, wide GEMMs (the SMPL-H blend): pairs of row tiles share the W tile by TMA multicast (cluster 1 x 2 x 1)
        if ((rc = make_map(h, &mw, g.W_hi, N, K, g.ldw, 64))) return rc;
        if ((rc = make_map(h, &mwl, g.W_lo, N, K, g.ldw, 64))) return rc;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((N + 127) / 128, (row_tiles + 1) & ~1, 1);      // an even number of row tiles (a tile past M loads zeros, stores nothing)
        cfg.blockDim = dim3(GEMM_THREADS); cfg.dynamicSmemBytes = Cfg<128>::SMEM_BYTES; cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 2; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        CUDA_TRY(h, cudaLaunchKernelEx(&cfg, gemm_split_f16_kernel<128, true>, ma, mw, mal, mwl, g.bias, g.res, g.ldr, g.C, g.C_hi, g.C_lo, g.ldc,
                                       M, N, K, g.epi, promote, (float*)nullptr, 0, 0, trace));
    } else if (wide) {
        if ((rc = make_map(h, &mw, g.W_hi, N, K, g.ldw, 128))) return rc;
        if ((rc = make_map(h, &mwl, g.W_lo, N, K, g.ldw, 128))) return rc;
        dim3 grid((N + 127) / 128, row_tiles, ksplit);
        idb_launch(g.pdl != 0, gemm_split_f16_kernel<128>, grid, GEMM_THREADS, Cfg<128>::SMEM_BYTES, st, ma, mw, mal, mwl, g.bias, g.res, g.ldr,
                   g.C, g.C_hi, g.C_lo, g.ldc, M, N, K, g.epi, promote, zero, g.zero_ld, g.zero_cols, trace);
    } else {
        if ((rc = make_map(h, &mw, g.W_hi, N, K, g.ldw, 64))) return rc;
        if ((rc = make_map(h, &mwl, g.W_lo, N, K, g.ldw, 64))) return rc;
        // at most one CTA per SM: the CTAs of a row tile split its column tiles, and a grid short of rows takes further row
        // tiles in turn (gemm_split_f16_persistent)
        const int col_tiles = (N + 63) / 64, sms = std::max(1, h->sm_count / ksplit);
        int cpr = col_tiles, gy = row_tiles;
        if (g_idb_gemm_persistent) {
            gy = std::min(row_tiles, sms);
            cpr = std::max(1, std::min(col_tiles, sms / row_tiles));
        }
        idb_launch(g.pdl != 0, gemm_split_f16_persistent, dim3(cpr, gy, ksplit), GEMM_THREADS, pers::SMEM_BYTES, st, ma, mw, mal, mwl, g.bias,
                   g.res, g.ldr, g.C, g.C_hi, g.C_lo, g.ldc, M, N, K, g.epi, promote, zero, g.zero_ld, g.zero_cols, trace);
    }
    LAUNCH_CHECK(h);
    return IDB_OK;
}

// Fused feed-forward block (see mlp_fused_kernel).  x / w1 / w2 as fp16 (hi, lo) pairs, row-major:
// x [M][256], w1 [F][256], w2 [256][F];  Z[M][256] = gelu(x w1^T + b1) w2^T + b2 + res, optionally followed by the layer's
// final LayerNorm (ln_w / ln_b) and an additional fp16 (hi, lo) copy of the output (Z_hi / Z_lo) for the next GEMM.
bool idb_mlp_wgmma_supported(int d_model, int d_ff) { return d_model == mlp::DM && d_ff == mlp::FC * mlp::CLUSTER; }

int idb_mlp_wgmma(idb_handle* h, const __half* x_hi, const __half* x_lo, const __half* w1_hi, const __half* w1_lo, const float* b1,
                    const __half* w2_hi, const __half* w2_lo, const float* b2, const float* res, int ldr, float* Z, int ldz, int M,
                    int pdl, cudaStream_t st, const float* ln_w, const float* ln_b, __half* Z_hi, __half* Z_lo) {
    long long* trace = g_idb_gemm_trace;
    g_idb_gemm_trace = nullptr;
    if (!(h->attr_mask & 2u)) {
        CUDA_TRY(h, cudaFuncSetAttribute(mlp_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mlp::SMEM_BYTES));
        h->attr_mask |= 2u;
    }
    const int F = mlp::FC * mlp::CLUSTER;
    CUtensorMap mx, mxl, mw1, mw1l, mw2, mw2l;
    int rc;
    if ((rc = make_map(h, &mx, x_hi, M, mlp::DM, mlp::DM, BM))) return rc;
    if ((rc = make_map(h, &mxl, x_lo, M, mlp::DM, mlp::DM, BM))) return rc;
    if ((rc = make_map(h, &mw1, w1_hi, F, mlp::DM, mlp::DM, mlp::FC))) return rc;
    if ((rc = make_map(h, &mw1l, w1_lo, F, mlp::DM, mlp::DM, mlp::FC))) return rc;
    // W2: boxes of 128 rows (one CTA's half of the output columns) x 64 hidden columns
    if ((rc = make_map(h, &mw2, w2_hi, mlp::DM, F, F, mlp::NH))) return rc;
    if ((rc = make_map(h, &mw2l, w2_lo, mlp::DM, F, F, mlp::NH))) return rc;
    dim3 grid(mlp::CLUSTER, (M + BM - 1) / BM);
    idb_launch(pdl != 0, mlp_fused_kernel, grid, NUM_THREADS, mlp::SMEM_BYTES, st, mx, mw1, mxl, mw1l, mw2, mw2l, b1, b2, res, ldr, Z, ldz, M, ln_w, ln_b, Z_hi, Z_lo, trace);
    LAUNCH_CHECK(h);
    return IDB_OK;
}
