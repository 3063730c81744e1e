// wgmma / TMA / mbarrier PTX wrappers and the fused feed-forward block as a device function, used by the kernels of
// gemm_wgmma.cu.  sm_90a only.
#pragma once
#include "common.cuh"

#include <cuda.h>

namespace tc {

constexpr int BM = 128;                // rows per CTA tile: two consumer warpgroups of 64 rows (one wgmma M each)
constexpr int BK = 64;                 // 64 fp16 = one 128-byte swizzle row
constexpr int MMA_K = 16;              // wgmma k per instruction for fp16 operands
constexpr int NUM_THREADS = 320;       // 8 consumer warps + TMA producer warp + exchange warp

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on the barrier at the same offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint32_t bar, uint32_t rank) {
    uint32_t rbar;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar) : "r"(bar), "r"(rank));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(rbar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// multicast variant: the box lands at the same shared-memory offset of every CTA in `mask` and completes on each one's barrier
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5}], [%2], %3;"
                 ::"r"(dst), "l"(map), "r"(bar), "h"(mask), "r"(c0), "r"(c1) : "memory");
}
// one lane of a fully active warp; the surrounding code stays warp-uniform
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}" : "=r"(pred));
    return pred != 0;
}

// K-major, SWIZZLE_128B canonical layout: rows of 128 B, 8-row groups 1024 B apart (wgmma matrix descriptor).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);     // start address  [0,14)
    d |= (uint64_t)1 << 16;                       // leading byte offset (16 B, unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;             // stride byte offset: 8 rows x 128 B
    d |= (uint64_t)1 << 62;                       // SWIZZLE_128B
    return d;
}

// ---- wgmma: D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, fp16 operands read from shared memory through descriptors, fp32
// accumulators in registers.  Thread (warp w of the warpgroup, lane l) holds, for j = 0 .. N/8 - 1:
//   d[4j], d[4j+1] = D[16w + l/4][8j + 2(l%4) + {0, 1}],   d[4j+2], d[4j+3] = the same columns of row + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define IDB_ACC8(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_f16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "
        "%27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
        "}"
        : IDB_ACC8(d, 0), IDB_ACC8(d, 8), IDB_ACC8(d, 16), IDB_ACC8(d, 24)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "
        "%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, "
        "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t"
        "}"
        : IDB_ACC8(d, 0), IDB_ACC8(d, 8), IDB_ACC8(d, 16), IDB_ACC8(d, 24), IDB_ACC8(d, 32), IDB_ACC8(d, 40), IDB_ACC8(d, 48), IDB_ACC8(d, 56)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
#undef IDB_ACC8

// One k-block (64 columns) of the split-precision product on this warpgroup's 64 rows:
//   small += A_lo W_hi^T + A_hi W_lo^T,   main (+)= A_hi W_hi^T        (descriptors of the k-block's first 16 columns)
template <int NR>
__device__ __forceinline__ void split_kblock(float (&main)[NR], float (&small)[NR], uint64_t dah, uint64_t dal, uint64_t dwh, uint64_t dwl,
                                             bool first_main, bool first_small, bool with_small = true) {
#pragma unroll
    for (int kk = 0; kk < BK / MMA_K; kk++) {
        const uint64_t koff = (uint64_t)((kk * MMA_K * 2) >> 4);   // +32 bytes per k-step in the start-address field
        if (with_small) {
            wgmma_f16(small, dal + koff, dwh + koff, (kk || !first_small) ? 1u : 0u);
            wgmma_f16(small, dah + koff, dwl + koff, 1u);
        }
        wgmma_f16(main, dah + koff, dwh + koff, (kk || !first_main) ? 1u : 0u);
    }
}

// ---------------------------------------------------------------------------------------------
// Fused feed-forward block  Z = gelu(X W1^T + b1) W2^T + b2 + R   for d_model 256, d_ff = 8 x 128.
//
// The two GEMMs of a decoder layer are each below one wave of work and their launches, prologues and the round trip of
// the fp16-pair intermediate cost more than the tensor work.  Here a cluster of 8 CTAs owns one 128-row tile: CTA j
// computes the 128-column chunk j of the hidden layer (GEMM 1, K = 256) into the registers of its two consumer
// warpgroups, which apply bias + GELU, split the result into (hi, lo) fp16 pairs and write them into shared memory
// directly in the K-major 128B-swizzled layout wgmma reads (S, one k-block of 64 hidden columns at a time).
//
// GEMM 2 runs on PAIRS of CTAs (j, j^1): as soon as a k-block of S is complete its owner also copies it into the
// partner's shared memory (cp.async.bulk shared::cta -> shared::cluster, completing on the partner's mbarrier) and each
// CTA of the pair multiplies BOTH hidden chunks (K = 256) with its HALF of the output columns (N = 128, CTA j owns
// columns 128 (j & 1) ..).  So only 4 instead of 8 partial products exist per output element and each is half as wide:
// the reduction that ends the kernel - CTA j PULLS rows 16j .. 16j+15 of the partials of both column halves over
// distributed shared memory and sums them in rank order (deterministic) - moves 56 KB per CTA instead of 112 KB.
// Then bias + residual, the layer's final LayerNorm, stores.
//
// Warp roles: warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of the tile: wgmma, GELU, reduction), warp 8 = TMA
// producer, warp 9 = exchange with the partner CTA.
//
// Shared memory (192 KB):  R0 [0, 64K)    GEMM 1 stage 0, then the partner's S (same layout as S)
//                          R1 [64K, 128K) GEMM 1 stage 1, then the W2 ring: 2 slots of 32 KB (k-block of 64: hi 16K | lo 16K)
//                          S  [128K,192K) S_hi [2][16K] | S_lo [2][16K]
//                          after GEMM 2: the fp32 partial tile [128][136] at offset 0.
namespace mlp {
constexpr int FC = 128;                       // hidden columns per CTA
constexpr int CLUSTER = 8;                    // d_ff / FC
constexpr int DM = 256;                       // d_model
constexpr int NH = DM / 2;                    // output columns per CTA in GEMM 2
constexpr int STAGE1 = 64 * 1024;             // A_hi 16K | W1_hi 16K | A_lo 16K | W1_lo 16K
constexpr int RING = 2 * STAGE1;
constexpr int S_BYTES = 64 * 1024;            // S_hi [2][16K] | S_lo [2][16K]
constexpr int W2SLOT = 32 * 1024;             // W2 k-block: hi [128 rows][128 B] | lo
constexpr int PLD = NH + 8;                   // fp32 partial row stride (floats): a half-warp's float2 stores (4 rows x 8
                                              // columns) fall on 32 distinct banks
constexpr int SMEM_BYTES = RING + S_BYTES + 1024 /*alignment slack*/ + 1024 /*barriers*/;
constexpr int CW = 8;                         // consumer warps
// barriers (8 B each, above the operand region): full1[2] 0,1 | empty1[2] 2,3 | gemm1_done 4 | w2full[2] 5,6 | s_ready[0] 7 |
// s_ready[1] 9 | w2empty[2] 10,11 | peer_free 12 | peer_s hi[2] 13,14 | peer_s lo[2] 15,16
}  // namespace mlp

__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

struct MlpArgs {
    const CUtensorMap *map_x, *map_w1, *map_xl, *map_w1l, *map_w2, *map_w2l;
    const float *b1, *b2, *res; int ldr;
    float* Z; int ldz;
    const float *ln_w, *ln_b;
    __half *Zh, *Zl;
};

// The feed-forward block of one 128-row tile on the cluster's 8 CTAs (see the comment above).  j = rank in the cluster =
// hidden chunk; m0 = first row of the tile; rows >= M are neither reduced nor stored.  Called by all 320 threads of the CTA
// (NUM_THREADS).
__device__ __forceinline__ void mlp_tile(uint8_t* smem_raw, const MlpArgs& a, int j, int m0, int M, long long* tr) {
    using namespace mlp;
    constexpr int NPASS = 1024 / (CW * 32);    // float4 elements of the 16 x 256 reduction slice per consumer thread
#define MTRACE(slot) do { if (tr) tr[slot] = clock64(); } while (0)
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bars = base + RING + S_BYTES;
    if (threadIdx.x == 0) {
        // The thread that initialises the barriers also requests the first two k-blocks of GEMM 1 at once - W1
        // (step-invariant), then, after the dependency wait, X - before the CTA barrier.  The two "operands landed" barriers
        // of GEMM 1 first, so that the first requests leave before the other barriers exist.
        mbar_init(bars, 1); mbar_init(bars + 8u, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int kb = 0; kb < 2; kb++) {
            const uint32_t dst = base + kb * STAGE1;
            mbar_arrive_expect_tx(bars + 8u * kb, STAGE1);
            tma_load_2d(dst + 16384, a.map_w1, bars + 8u * kb, kb * BK, j * FC);
            tma_load_2d(dst + 49152, a.map_w1l, bars + 8u * kb, kb * BK, j * FC);
        }
        pdl_wait();
        chain_mark(2, 1);
        for (int kb = 0; kb < 2; kb++) {
            const uint32_t dst = base + kb * STAGE1;
            tma_load_2d(dst, a.map_x, bars + 8u * kb, kb * BK, m0);
            tma_load_2d(dst + 32768, a.map_xl, bars + 8u * kb, kb * BK, m0);
        }
        for (int s = 0; s < 2; s++) {
            mbar_init(bars + 8u * (2 + s), CW); mbar_init(bars + 8u * (5 + s), 1); mbar_init(bars + 8u * (10 + s), CW);
            mbar_init(bars + 8u * (13 + s), 1); mbar_init(bars + 8u * (15 + s), 1);
        }
        mbar_init(bars + 8u * 4, CW);
        mbar_init(bars + 8u * 7, CW * 32); mbar_init(bars + 8u * 9, CW * 32);
        mbar_init(bars + 8u * 12, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // the partner's copies of its S k-blocks complete on these four (16 KB each: hi / lo of a k-block)
        for (int s = 0; s < 4; s++) mbar_arrive_expect_tx(bars + 8u * (13 + s), 16384u);
        asm volatile("prefetch.tensormap [%0];" ::"l"(a.map_w2) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(a.map_w2l) : "memory");
    }
    __syncthreads();

    const CUtensorMap& map_x = *a.map_x; const CUtensorMap& map_w1 = *a.map_w1; const CUtensorMap& map_xl = *a.map_xl;
    const CUtensorMap& map_w1l = *a.map_w1l; const CUtensorMap& map_w2 = *a.map_w2; const CUtensorMap& map_w2l = *a.map_w2l;
    const float* __restrict__ b1 = a.b1; const float* __restrict__ b2 = a.b2; const float* __restrict__ res = a.res;
    const int ldr = a.ldr, ldz = a.ldz;
    float* __restrict__ Z = a.Z; const float* __restrict__ ln_w = a.ln_w; const float* __restrict__ ln_b = a.ln_b;
    __half* __restrict__ Zh = a.Zh; __half* __restrict__ Zl = a.Zl;
    uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t s_base = base + RING;
    auto bar_full1 = [&](int s) { return bars + 8u * s; };
    auto bar_empty1 = [&](int s) { return bars + 8u * (2 + s); };
    const uint32_t bar_g1done = bars + 8u * 4;
    auto bar_w2full = [&](int s) { return bars + 8u * (5 + s); };
    auto bar_sready = [&](int kb) { return bars + 8u * (kb ? 9 : 7); };
    auto bar_w2empty = [&](int s) { return bars + 8u * (10 + s); };
    const uint32_t bar_peer_free = bars + 8u * 12;
    auto bar_peer_s = [&](int kb, int lo) { return bars + 8u * (13 + 2 * lo + kb); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int jp = j ^ 1, hcol = j & 1;          // partner CTA (same pair of hidden chunks), this CTA's half of the output columns
    const bool consumer = warp < CW;
    if (threadIdx.x == 0) MTRACE(1);

    // Every CTA's barriers must exist (above) before a partner arrives on them or copies into this CTA's shared memory:
    // one cluster barrier, arrive here, wait where each role first needs it (the consumers only after GEMM 1), so that its
    // latency stays off the critical path.
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");      // (the fence.mbarrier_init above is the release)
#define CLUSTER_WAIT() asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory")

    float4 o[NPASS];                     // this thread's elements of the closing reduction (consumers)
    if (warp == CW) {
        // ===================== TMA producer =====================
        for (int kb = 2; kb < 4; kb++) {
            const int s = kb & 1;
            mbar_wait(bar_empty1(s), 0);
            const uint32_t dst = base + s * STAGE1;
            if (elect_one()) {
                mbar_arrive_expect_tx(bar_full1(s), STAGE1);
                tma_load_2d(dst, &map_x, bar_full1(s), kb * BK, m0);
                tma_load_2d(dst + 16384, &map_w1, bar_full1(s), kb * BK, j * FC);
                tma_load_2d(dst + 32768, &map_xl, bar_full1(s), kb * BK, m0);
                tma_load_2d(dst + 49152, &map_w1l, bar_full1(s), kb * BK, j * FC);
            }
            __syncwarp();
        }
        CLUSTER_WAIT();
        // GEMM 1 finished reading the ring: stream this CTA's half of W2's rows (output columns 128 hcol ..) for the pair's
        // 256 hidden columns through the two 32 KB slots of R1, in the order GEMM 2 consumes them: own chunk j (its S is
        // local), then the partner's
        mbar_wait(bar_g1done, 0);
        for (int i = 0; i < 4; i++) {
            const int sl = i & 1;
            if (i >= 2) mbar_wait(bar_w2empty(sl), 0);
            if (elect_one()) {
                const uint32_t dst = base + STAGE1 + sl * W2SLOT;
                const int kcol = (i < 2 ? j : jp) * FC + (i & 1) * BK;
                mbar_arrive_expect_tx(bar_w2full(sl), W2SLOT);
                tma_load_2d(dst, &map_w2, bar_w2full(sl), kcol, hcol * NH);
                tma_load_2d(dst + 16384, &map_w2l, bar_w2full(sl), kcol, hcol * NH);
            }
            __syncwarp();
        }
    } else if (warp == CW + 1) {
        // ===================== exchange with the partner CTA =====================
        CLUSTER_WAIT();
        // GEMM 1 complete: R0 may now receive the partner's S (tell it so), and this CTA may copy into the partner's once it says
        // the same
        mbar_wait(bar_g1done, 0);
        if (elect_one()) mbar_arrive_remote(bar_peer_free, jp);
        __syncwarp();
        for (int kb = 0; kb < 2; kb++) {
            mbar_wait(bar_sready(kb), 0);        // all consumer threads have written (and proxy-fenced) this k-block of S
            if (kb == 0) mbar_wait(bar_peer_free, 0);
            if (elect_one()) {
                uint32_t rdst, rbar_hi, rbar_lo;
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rdst) : "r"(base + kb * 16384), "r"(jp));
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar_hi) : "r"(bar_peer_s(kb, 0)), "r"(jp));
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar_lo) : "r"(bar_peer_s(kb, 1)), "r"(jp));
                asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(rdst), "r"(s_base + kb * 16384), "r"(16384u), "r"(rbar_hi) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(rdst + 32768u), "r"(s_base + 32768 + kb * 16384), "r"(16384u), "r"(rbar_lo) : "memory");
            }
            __syncwarp();
        }
    } else {
        // ===================== consumer warpgroups =====================
        const int wg = warp >> 2;                                    // rows 64 wg .. of the tile
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // this thread's accumulator rows: r0 and r0 + 8
        const int cq = 2 * (lane & 3);                               // ... and columns 8 j + cq, + 1
        const uint32_t a_off = (uint32_t)wg * 8192u;                 // the warpgroup's 64 rows of a 128-row operand tile
        {
            // ---- GEMM 1: hidden chunk [128 x 128] = X [128 x 256] . W1[chunk j]^T
            float acc[64], accs[64];
            for (int kb = 0; kb < 4; kb++) {
                const int s = kb & 1;
                mbar_wait(bar_full1(s), (kb >> 1) & 1);
                if (kb == 0 && threadIdx.x == 0) MTRACE(2);
                const uint32_t st = base + s * STAGE1;
                wgmma_fence();
                split_kblock(acc, accs, make_smem_desc(st + a_off), make_smem_desc(st + 32768 + a_off), make_smem_desc(st + 16384),
                             make_smem_desc(st + 49152), kb == 0, kb == 0);
                wgmma_commit();
                wgmma_wait0();
                __syncwarp();
                if (lane == 0) { mbar_arrive(bar_empty1(s)); if (kb == 3) mbar_arrive(bar_g1done); }
            }
            if (threadIdx.x == 0) MTRACE(3);
            CLUSTER_WAIT();
            pdl_wait();
            // ---- bias + GELU -> (hi, lo) fp16 pairs in the swizzled K-major A layout, one k-block of S (64 hidden columns) at a
            // time, so that GEMM 2 and the copy to the partner can start on the first while the second is produced
#pragma unroll
            for (int kb = 0; kb < 2; kb++) {
#pragma unroll
                for (int jj = 0; jj < 8; jj++) {
                    const int jx = kb * 8 + jj;
                    const float2 bb = *reinterpret_cast<const float2*>(b1 + j * FC + 8 * jx + cq);
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) {
                        const int r = r0 + 8 * hh;
                        uint32_t hw, lw;
                        gelu_split_x2(acc[4 * jx + 2 * hh], acc[4 * jx + 2 * hh + 1], accs[4 * jx + 2 * hh], accs[4 * jx + 2 * hh + 1], bb, hw, lw);
                        uint8_t* p = base_ptr + RING + kb * 16384 + r * 128 + ((jj ^ (r & 7)) * 16) + cq * 2;
                        *reinterpret_cast<uint32_t*>(p) = hw;
                        *reinterpret_cast<uint32_t*>(p + 32768) = lw;
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy S writes -> visible to wgmma and the bulk copy
                mbar_arrive(bar_sready(kb));
            }
            if (threadIdx.x == 0) MTRACE(5);
        }
        {
            // ---- GEMM 2: [128 x 128] (this CTA's half of the output columns) = S_pair [128 x 256] . W2[half rows, pair's 256 columns]^T.
            // A = S k-blocks (own, then the partner's copied into R0), B = W2 k-blocks in the R1 ring.  Order of the additions per
            // accumulator: own chunk, then the partner's, k ascending - fixed per CTA, independent of M.
            float acc[64], accs[64];
            for (int i = 0; i < 4; i++) {
                const int sl = i & 1, kb = i & 1;
                uint32_t a_hi;
                if (i < 2) {
                    mbar_wait(bar_sready(kb), 0);
                    a_hi = s_base + kb * 16384;
                } else {
                    mbar_wait(bar_peer_s(kb, 0), 0);
                    mbar_wait(bar_peer_s(kb, 1), 0);
                    a_hi = base + kb * 16384;
                }
                mbar_wait(bar_w2full(sl), (i >> 1) & 1);
                const uint32_t w2 = base + STAGE1 + sl * W2SLOT;
                wgmma_fence();
                split_kblock(acc, accs, make_smem_desc(a_hi + a_off), make_smem_desc(a_hi + 32768 + a_off), make_smem_desc(w2),
                             make_smem_desc(w2 + 16384), i == 0, i == 0);
                wgmma_commit();
                wgmma_wait0();
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_w2empty(sl));
            }
            if (threadIdx.x == 0) MTRACE(8);
            // both warpgroups have finished reading the operand buffers: they become the fp32 partial tile
            asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
            for (int jx = 0; jx < 16; jx++)
#pragma unroll
                for (int hh = 0; hh < 2; hh++)
                    *reinterpret_cast<float2*>(reinterpret_cast<float*>(base_ptr) + (size_t)(r0 + 8 * hh) * PLD + 8 * jx + cq) =
                        make_float2(fmaf(accs[4 * jx + 2 * hh], 1.0f / 2048.0f, acc[4 * jx + 2 * hh]),
                                    fmaf(accs[4 * jx + 2 * hh + 1], 1.0f / 2048.0f, acc[4 * jx + 2 * hh + 1]));
            if (threadIdx.x == 0) MTRACE(9);
        }
    }
#undef CLUSTER_WAIT
    // ===================== cross-CTA reduction over distributed shared memory =====================
    // Every CTA has written its [128 x 128] fp32 partial product (its half of the output columns, its pair's 256 hidden columns)
    // into its own (now idle) operand region; after a cluster barrier CTA j PULLS rows 16j .. 16j+15 of all 8 partials - 4 per
    // column half - with coalesced 16-byte remote loads and sums each half's four in rank order (56 KB per CTA over the SM-to-SM
    // network).  One WARP per row (rows warp, warp + 8): pass t of a lane is row warp + 8 (t >> 1), column half t & 1, columns
    // 128 (t & 1) + 4 lane .. + 3 - so a warp instruction reads or writes 512 contiguous bytes and the row's LayerNorm
    // statistics are warp sums (no shared memory, no block barrier).
    __syncwarp();
    cluster_sync_all();                  // every CTA's partial tile is complete and visible cluster-wide
    if (threadIdx.x == 0) MTRACE(10);
    if (consumer) {
#pragma unroll
        for (int t = 0; t < NPASS; t++) {
            const int rr = warp + CW * (t >> 1), hh = t & 1;      // column half hh: its partials live in CTAs hh, hh + 2, hh + 4, hh + 6
            const int row = m0 + j * 16 + rr, c4 = hh * 32 + lane;
            const uint32_t off = base + (uint32_t)(((j * 16 + rr) * PLD + lane * 4) * 4);   // same offset in every CTA of the cluster
            float4 p[CLUSTER / 2];
#pragma unroll
            for (int i = 0; i < CLUSTER / 2; i++) {
                uint32_t ra;
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(off), "r"(2 * i + hh));
                asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(p[i].x), "=f"(p[i].y), "=f"(p[i].z), "=f"(p[i].w) : "r"(ra));
            }
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 0; i < CLUSTER / 2; i++) {      // rank order: deterministic
                acc.x += p[i].x; acc.y += p[i].y; acc.z += p[i].z; acc.w += p[i].w;
            }
            o[t] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row < M) {
                const float4 bb = *reinterpret_cast<const float4*>(b2 + c4 * 4);
                const float4 r4 = __ldcg(reinterpret_cast<const float4*>(res + (size_t)row * ldr + c4 * 4));
                o[t] = make_float4((acc.x + bb.x) + r4.x, (acc.y + bb.y) + r4.y, (acc.z + bb.z) + r4.z, (acc.w + bb.w) + r4.w);
            }
        }
        // this thread's remote reads are complete (their values were consumed above): arrive on the closing cluster barrier now,
        // wait for it after the LayerNorm and the stores (the operands tie the instruction to the sums of every pass)
        asm volatile("barrier.cluster.arrive.release.aligned;" ::"f"(o[0].x), "f"(o[1].x), "f"(o[NPASS - 2].x), "f"(o[NPASS - 1].x) : "memory");
        if (ln_w) {
            // the layer's final LayerNorm, fused: a row = the two passes 2g, 2g + 1 of one warp
            const float4 w0 = *reinterpret_cast<const float4*>(ln_w + lane * 4), w1 = *reinterpret_cast<const float4*>(ln_w + 128 + lane * 4);
            const float4 b0 = *reinterpret_cast<const float4*>(ln_b + lane * 4), b1v = *reinterpret_cast<const float4*>(ln_b + 128 + lane * 4);
#pragma unroll
            for (int g = 0; g < NPASS / 2; g++) {
                float4& oa = o[2 * g]; float4& ob = o[2 * g + 1];
                const float mean = warp_sum(((oa.x + oa.y) + (oa.z + oa.w)) + ((ob.x + ob.y) + (ob.z + ob.w))) * (1.0f / DM);
                oa.x -= mean; oa.y -= mean; oa.z -= mean; oa.w -= mean; ob.x -= mean; ob.y -= mean; ob.z -= mean; ob.w -= mean;
                const float sq = warp_sum(((oa.x * oa.x + oa.y * oa.y) + (oa.z * oa.z + oa.w * oa.w)) + ((ob.x * ob.x + ob.y * ob.y) + (ob.z * ob.z + ob.w * ob.w)));
                const float rstd = 1.0f / sqrtf(sq * (1.0f / DM) + 1e-5f);
                oa = make_float4(oa.x * rstd * w0.x + b0.x, oa.y * rstd * w0.y + b0.y, oa.z * rstd * w0.z + b0.z, oa.w * rstd * w0.w + b0.w);
                ob = make_float4(ob.x * rstd * w1.x + b1v.x, ob.y * rstd * w1.y + b1v.y, ob.z * rstd * w1.z + b1v.z, ob.w * rstd * w1.w + b1v.w);
            }
        }
#pragma unroll
        for (int t = 0; t < NPASS; t++) {
            const int rr = warp + CW * (t >> 1), c4 = (t & 1) * 32 + lane;
            const int row = m0 + j * 16 + rr;
            if (row < M) {
                *reinterpret_cast<float4*>(Z + (size_t)row * ldz + c4 * 4) = o[t];
                if (Zh) {
                    __half2 h01, h23, l01, l23;
                    split_f16x2(o[t].x, o[t].y, h01, l01);
                    split_f16x2(o[t].z, o[t].w, h23, l23);
                    *reinterpret_cast<uint2*>(Zh + (size_t)row * ldz + c4 * 4) = make_uint2(*reinterpret_cast<uint32_t*>(&h01), *reinterpret_cast<uint32_t*>(&h23));
                    *reinterpret_cast<uint2*>(Zl + (size_t)row * ldz + c4 * 4) = make_uint2(*reinterpret_cast<uint32_t*>(&l01), *reinterpret_cast<uint32_t*>(&l23));
                }
            }
        }
        if (threadIdx.x == 0) MTRACE(11);
    } else {
        asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    }
    __syncwarp();
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");      // nobody leaves (and frees / reuses its shared memory) while peers still read it
    if (threadIdx.x == 0) MTRACE(12);
    __syncthreads();
#undef MTRACE
}

}  // namespace tc
