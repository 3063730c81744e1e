// Micro-benchmark of the cross-CTA exchange of the feed-forward cluster kernel (8-CTA clusters, one CTA per SM, all
// 15 clusters exchanging at once): every CTA must end up with 7 remote blocks of BLK bytes.
//   mode 0: pull with ld.shared::cluster.v4 (what tc_mlp.cuh does), 512 threads
//   mode 1: push with cp.async.bulk.shared::cluster.shared::cta (TMA engine), completion on the receiver's mbarrier
//   mode 2: push with st.async (remote store + complete_tx on the receiver's mbarrier), 512 threads
//   mode 3: like 1, the 7 blocks cut into 4 pieces each (28 bulk copies per CTA)
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o interdiff_b200/build/dsmem_bench profiles/dsmem_bench.cu
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>
#include <cuda_runtime.h>

constexpr int CL = 8, BLK = 14 * 1024, NT = 512;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t a, int r) {
    uint32_t o; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(o) : "r"(a), "r"(r)); return o;
}

__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(NT, 1) k_exchange(int mode, long long* out, float* sink) {
    extern __shared__ __align__(1024) uint8_t sm[];
    uint8_t* send = sm;                       // [CL][BLK]   block i goes to CTA i
    uint8_t* recv = sm + CL * BLK;            // [CL][BLK]   slot i comes from CTA i (mode 0 reads the peers' send buffers instead)
    uint64_t* bar = reinterpret_cast<uint64_t*>(sm + 2 * CL * BLK);
    uint32_t rank; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const int tid = threadIdx.x;
    for (int i = tid; i < CL * BLK / 4; i += NT) reinterpret_cast<float*>(send)[i] = (float)(i + rank);
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"((CL - 1) * BLK) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    cluster_sync_all();
    const long long t0 = clock64();
    float acc = 0.f;
    if (mode == 0) {
        for (int idx = tid; idx < BLK / 16; idx += NT) {
            float4 p[CL];
#pragma unroll
            for (int i = 0; i < CL; i++) {
                const uint32_t ra = mapa(smem_u32(send + rank * BLK + idx * 16), i);
                asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(p[i].x), "=f"(p[i].y), "=f"(p[i].z), "=f"(p[i].w) : "r"(ra));
            }
#pragma unroll
            for (int i = 0; i < CL; i++) acc += p[i].x + p[i].y + p[i].z + p[i].w;
        }
    } else if (mode == 1 || mode == 3) {
        const int pieces = mode == 3 ? 4 : 1, pb = BLK / pieces;
        if (tid < (CL - 1) * pieces) {
            const int i = (rank + 1 + tid / pieces) % CL, pc = tid % pieces;      // staggered peers
            const uint32_t dst = mapa(smem_u32(recv + rank * BLK + pc * pb), i), rbar = mapa(smem_u32(bar), i);
            asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "r"(smem_u32(send + i * BLK + pc * pb)), "r"(pb), "r"(rbar) : "memory");
        }
        uint32_t ok = 0;
        while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(0) : "memory");
        for (int idx = tid; idx < BLK / 16; idx += NT) {
#pragma unroll
            for (int i = 0; i < CL; i++) {
                const float4 p = *reinterpret_cast<const float4*>((i == (int)rank ? send : recv) + i * BLK + idx * 16);
                acc += p.x + p.y + p.z + p.w;
            }
        }
    } else {
        for (int k = 1; k < CL; k++) {
            const int i = (rank + k) % CL;
            const uint32_t rbar = mapa(smem_u32(bar), i);
            for (int idx = tid; idx < BLK / 16; idx += NT) {
                const float4 v = *reinterpret_cast<const float4*>(send + i * BLK + idx * 16);
                const uint32_t dst = mapa(smem_u32(recv + rank * BLK + idx * 16), i);
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
                             ::"r"(dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(rbar) : "memory");
            }
        }
        uint32_t ok = 0;
        while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(0) : "memory");
        for (int idx = tid; idx < BLK / 16; idx += NT) {
#pragma unroll
            for (int i = 0; i < CL; i++) {
                const float4 p = *reinterpret_cast<const float4*>((i == (int)rank ? send : recv) + i * BLK + idx * 16);
                acc += p.x + p.y + p.z + p.w;
            }
        }
    }
    __syncthreads();
    const long long t1 = clock64();
    cluster_sync_all();
    const long long t2 = clock64();
    if (acc == 1.2345f) *sink = acc;
    if (tid == 0) { out[2 * blockIdx.x] = t1 - t0; out[2 * blockIdx.x + 1] = t2 - t0; }
}

int main() {
    const int nclusters = 15, nb = nclusters * CL, smem = 2 * CL * BLK + 64;
    cudaFuncSetAttribute(k_exchange, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    long long* out; float* sink;
    cudaMalloc(&out, nb * 2 * sizeof(long long)); cudaMalloc(&sink, 4);
    const char* names[4] = {"pull ld.shared::cluster", "push cp.async.bulk (7 copies)", "push st.async", "push cp.async.bulk (28 copies)"};
    for (int mode = 0; mode < 4; mode++) {
        std::vector<long long> h(nb * 2), a, b;
        for (int rep = 0; rep < 5; rep++) {
            k_exchange<<<nb, NT, smem>>>(mode, out, sink);
            if (cudaDeviceSynchronize() != cudaSuccess) { printf("mode %d failed: %s\n", mode, cudaGetErrorString(cudaGetLastError())); return 1; }
            cudaMemcpy(h.data(), out, nb * 2 * sizeof(long long), cudaMemcpyDeviceToHost);
            if (rep >= 2) for (int i = 0; i < nb; i++) { a.push_back(h[2 * i]); b.push_back(h[2 * i + 1]); }
        }
        std::sort(a.begin(), a.end()); std::sort(b.begin(), b.end());
        printf("%-32s %d B per peer: data in registers median %lld max %lld cycles; + cluster barrier median %lld max %lld  (%.1f B/clk/SM incoming)\n",
               names[mode], BLK, a[a.size() / 2], a.back(), b[b.size() / 2], b.back(), 7.0 * BLK / a[a.size() / 2]);
    }
    return 0;
}
