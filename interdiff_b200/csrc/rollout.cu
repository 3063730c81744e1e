// Autoregressive rollout (SURVEY 8f rank 2, BASELINE configs[4]): the step between two sampling windows of
// reference eval_smpl_long.py:247-285 on the device - `get_batch` (:26-84) re-canonicalises the last past_len predicted
// frames into the next window's inputs, `denormalize` (:278) maps a window's outputs back to world coordinates.
//
// What the reference does, and what it leaves undefined: get_batch keeps `rotation` = identity (:39-40) and takes the
// pelvis of the FIRST of the past_len frames as `centroid` (:38), so the re-canonicalisation is a per-sample translation:
// body / object translations minus the centroid (:43-46, :58-59), rotations unchanged (:52-55, :60-64), and the
// future_len inputs are copies of the last past frame (:78).  The new window's gt tensor is then rebuilt by
// MDM._get_embeddings (model/diffusion_smpl.py:195-214): axis-angle -> matrix -> first two rows.  `denormalize` and
// `correct` are called but never defined upstream (:278, :285); here denormalize is the exact inverse of get_batch (add
// the accumulated centroid to every translation / vertex / joint) and correct is the identity.  Upstream get_batch
// cannot execute for any batch size (`.unsqueeze(0).repeat(B, 1)` on a (B,3) tensor raises), so this row is restated
// intent: parity is pinned to oracle/restate.py::rollout_next_window only (DESIGN.md "Oracle").
#include "common.cuh"
#include "rot.cuh"

namespace {

// body (T,B,Db): [66 axis-angle | 90 hand | 3 trans] (Db = 159), obj (T,B,6): [axis-angle | trans], jtr (T,B,J,3).
// gt_out (B,1,144,T): frames t < past from source frame T - past + t, frames >= past = copies of frame past - 1.
__global__ void __launch_bounds__(128)
k_rollout_next(const float* __restrict__ body, const float* __restrict__ obj, const float* __restrict__ jtr, float* __restrict__ gt_out,
               float* __restrict__ centroid_out, int T, int B, int J, int Db, int past) {
    __shared__ float s_c[3];
    __shared__ float s_f[16][144];          // the past frames' channel vectors (past <= 16)
    const int b = blockIdx.x, tid = threadIdx.x;
    if (tid < 3) {
        s_c[tid] = jtr[(((size_t)(T - past) * B + b) * J + 0) * 3 + tid];      // pelvis of the first past frame
        centroid_out[(size_t)b * 3 + tid] = s_c[tid];
    }
    __syncthreads();
    for (int i = tid; i < past * 23; i += 128) {
        const int t = i / 23, j = i % 23, src = T - past + t;
        const float* aa = j < 22 ? body + ((size_t)src * B + b) * Db + j * 3 : obj + ((size_t)src * B + b) * 6;
        float R[9];
        idb_axis_angle_to_matrix(aa, R);
        float* dst = s_f[t] + (j < 22 ? j * 6 : 135);
        for (int e = 0; e < 6; e++) dst[e] = R[e];                             // matrix_to_rotation_6d: the first two ROWS
    }
    for (int i = tid; i < past * 6; i += 128) {
        const int t = i / 6, e = i % 6, src = T - past + t;
        if (e < 3) s_f[t][132 + e] = body[((size_t)src * B + b) * Db + (Db - 3) + e] - s_c[e];
        else s_f[t][141 + e - 3] = obj[((size_t)src * B + b) * 6 + e] - s_c[e - 3];
    }
    __syncthreads();
    for (int i = tid; i < 144 * T; i += 128) {
        const int c = i / T, t = i % T;
        gt_out[((size_t)b * 144 + c) * T + t] = s_f[t < past ? t : past - 1][c];
    }
}

// x[(t*B + b) * ld + col0 + k*3 + c] += sign * offset[b*3 + c]   for k < K
__global__ void k_add_offset(float* __restrict__ x, long long ld, int col0, int K, int T, int B, const float* __restrict__ offset, float sign) {
    const long long n = (long long)T * B * K * 3;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % 3);
        const long long r = i / 3 / K;               // t*B + b
        const int k = (int)((i / 3) % K), b = (int)(r % B);
        x[r * ld + col0 + (long long)k * 3 + c] += sign * offset[b * 3 + c];
    }
}

}  // namespace

extern "C" int idb_rollout_next_window(idb_handle* h, int T, int B, int J, int Db, int past_len, const float* body, const float* obj,
                                       const float* jtr, float* gt_out, float* centroid_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !body || !obj || !jtr || !gt_out || !centroid_out) return IDB_ERR_ARG;
    if (T <= 0 || B <= 0 || J <= 0 || Db < 69 || past_len < 1 || past_len > 16 || past_len > T)
        return idb_fail(h, IDB_ERR_ARG, "rollout: 1 <= past_len <= min(16, T), body rows of >= 69 channels");
    k_rollout_next<<<B, 128, 0, (cudaStream_t)stream>>>(body, obj, jtr, gt_out, centroid_out, T, B, J, Db, past_len);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

extern "C" int idb_add_offset(idb_handle* h, int T, int B, int K, long long ld, int col0, float* x, const float* offset, float sign,
                              void* stream) {
    IDB_ENTER(h);
    if (!h || !x || !offset || T <= 0 || B <= 0 || K <= 0 || ld < (long long)col0 + 3LL * K) return IDB_ERR_ARG;
    const long long n = (long long)T * B * K * 3;
    const int blocks = (int)((n + 255) / 256 < 132 * 8 ? (n + 255) / 256 : 132 * 8);
    k_add_offset<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, ld, col0, K, T, B, offset, sign);
    LAUNCH_CHECK(h);
    return IDB_OK;
}
