// Token stage of the skeleton model's conditioning encoder (idb_encode_condition_skeleton in denoiser.cu, which runs the
// shared encoder layers on its output).
#include "common.cuh"

namespace {

constexpr int D = 256;    // d_model (checked at idb_denoiser_init)

// Skeleton model (model/diffusion_skeleton.py:204-212).  body (>=Tp,B,Cb), obj (>=Tp,B,Co) sequence-first: frame t of
// sample b is row t*B + b, so the first Tp frames are read in place.  Per sample b: token pairs [b*Tp+t][Cp] = [body | obj | 0]
// and addend[b*Tp+t][:] = (shapeEmbedding(zero_pose_obj[b]) + b_body + b_obj) + pe[t], the shape embedding in fp32.
__global__ void k_cond_tokens_skeleton(const float* __restrict__ body, const float* __restrict__ obj, const float* __restrict__ zp,
                                       const float* __restrict__ ws, const float* __restrict__ bs, const float* __restrict__ b_in,
                                       const float* __restrict__ pe, __half* __restrict__ xtok_b, __half* __restrict__ xtok_s,
                                       float* __restrict__ add, int B, int Tp, int Cb, int Co, int Cp) {
    __shared__ __align__(16) float s_shp[D];
    __shared__ float s_zp[IDB_SHAPE_EMB_MAX_IN];
    const int b = blockIdx.x;
    for (int k = threadIdx.x; k < Co; k += blockDim.x) s_zp[k] = zp[(size_t)b * Co + k];
    __syncthreads();
    for (int n = threadIdx.x; n < D; n += blockDim.x) {
        float acc = 0.f;
        for (int k = 0; k < Co; k++) acc = fmaf(ws[(size_t)n * Co + k], s_zp[k], acc);
        s_shp[n] = acc + bs[n];
    }
    for (int i = threadIdx.x; i < Tp * Cp; i += blockDim.x) {
        const int t = i / Cp, c = i % Cp;
        const size_t row = (size_t)t * B + b;
        const float v = c < Cb ? body[row * Cb + c] : c < Cb + Co ? obj[row * Co + (c - Cb)] : 0.f;
        const size_t o = ((size_t)b * Tp + t) * Cp + c;
        split_f16(v, xtok_b[o], xtok_s[o]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < Tp * (D / 4); i += blockDim.x) {
        const int t = i / (D / 4), c4 = i % (D / 4);
        const float4 p = reinterpret_cast<const float4*>(s_shp)[c4], bi = reinterpret_cast<const float4*>(b_in)[c4];
        const float4 q = reinterpret_cast<const float4*>(pe + (size_t)t * D)[c4];
        reinterpret_cast<float4*>(add + ((size_t)b * Tp + t) * D)[c4] =
            make_float4((p.x + bi.x) + q.x, (p.y + bi.y) + q.y, (p.z + bi.z) + q.z, (p.w + bi.w) + q.w);
    }
}

}  // namespace

void idb_cond_tokens_skeleton(const float* body, const float* obj, const float* zero_pose_obj, const float* w_shape, const float* b_shape,
                              const float* b_in, const float* pe, __half* xtok_b, __half* xtok_s, float* add, int B, int Tp, int Cb, int Co,
                              int Cp, cudaStream_t st) {
    k_cond_tokens_skeleton<<<B, 256, 0, st>>>(body, obj, zero_pose_obj, w_shape, b_shape, b_in, pe, xtok_b, xtok_s, add, B, Tp, Cb, Co, Cp);
}
