// SMPL-H linear blend skinning (fp32).  Replaces reference
// libsmpl/smplpytorch/pytorch/smpl_layer.py:72-175, rodrigues_layer.py:13-52, tensutils.py:6-53.
//
// Data layout in HBM (built once in idb_body_init):
//   posedirsT  [Kp][3][V]   k-major so a warp reads 32 consecutive vertices of one basis row
//   shapedirsT [NB][3][V]
//   v_templT   [3][V]
//   weightsT   [J][V]
//   J_templ [J][3], J_shape [J][3][NB]: the joint regressor folded through the shape blend,
//     J_rest = J_reg (v_t + S beta) = J_reg v_t + (J_reg S) beta   (exact algebra, computed in
//     float64 on the host; the reference evaluates the left form in fp32)
// Two kernels per call:
//   k_lbs_pose  (one block per frame): Rodrigues (quaternion route), rest joints, kinematic chain,
//               A_j = G_j - [0 | G_j J_j], pose_map = vec(R_1..R_{J-1} - I)
//   k_lbs_skin  (vertex tile x frame group): v_posed = v_t + S beta + P pose_map; T = sum_j w_j A_j;
//               verts = T [v_posed; 1] + trans.  Each block keeps FB frames of pose_map / A in
//               shared memory and streams the bases once for all of them.
#include "common.cuh"
#include "body.cuh"

namespace {

constexpr int FB = 16;  // frames per skinning block

__global__ void k_lbs_pose(const float* __restrict__ pose, const float* __restrict__ betas, const float* __restrict__ trans,
                           const float* __restrict__ J_templ, const float* __restrict__ J_shape,
                           const int* __restrict__ parents, float* __restrict__ Aout, float* __restrict__ pose_map,
                           float* __restrict__ jtr, int J, int NB, int Kp, __half* __restrict__ pm_hi, __half* __restrict__ pm_lo, int Kld,
                           const int* __restrict__ depth, int max_depth) {
    extern __shared__ float sm[];
    float* sR = sm;            // [J][9]
    float* sJ = sR + J * 9;    // [J][3]
    float* sG = sJ + J * 3;    // [J][12]
    const int f = blockIdx.x, j = threadIdx.x;
    if (j < J) {
        // batch_rodrigues (rodrigues_layer.py:41-52): angle = |aa + 1e-8|
        const float ax = pose[(size_t)f * J * 3 + j * 3 + 0], ay = pose[(size_t)f * J * 3 + j * 3 + 1], az = pose[(size_t)f * J * 3 + j * 3 + 2];
        const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
        const float angle = sqrtf(bx * bx + by * by + bz * bz);
        const float nx = ax / angle, ny = ay / angle, nz = az / angle;
        const float half = angle * 0.5f;
        const float c = cosf(half), s = sinf(half);
        float qw = c, qx = s * nx, qy = s * ny, qz = s * nz;
        const float qn = sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
        qw /= qn; qx /= qn; qy /= qn; qz /= qn;
        const float w2 = qw * qw, x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
        const float wx = qw * qx, wy = qw * qy, wz = qw * qz, xy = qx * qy, xz = qx * qz, yz = qy * qz;
        float* R = sR + j * 9;
        R[0] = w2 + x2 - y2 - z2; R[1] = 2 * xy - 2 * wz;   R[2] = 2 * wy + 2 * xz;
        R[3] = 2 * wz + 2 * xy;   R[4] = w2 - x2 + y2 - z2; R[5] = 2 * yz - 2 * wx;
        R[6] = 2 * xz - 2 * wy;   R[7] = 2 * wx + 2 * yz;   R[8] = w2 - x2 - y2 + z2;
        for (int c3 = 0; c3 < 3; c3++) {
            float v = J_templ[j * 3 + c3];
            for (int b = 0; b < NB; b++) v = fmaf(J_shape[(j * 3 + c3) * NB + b], betas[(size_t)f * NB + b], v);
            sJ[j * 3 + c3] = v;
        }
        if (j >= 1)
            for (int e = 0; e < 9; e++) {
                const float pm = R[e] - ((e == 0 || e == 4 || e == 8) ? 1.0f : 0.0f);
                if (pm_hi) split_f16(pm, pm_hi[(size_t)f * Kld + (j - 1) * 9 + e], pm_lo[(size_t)f * Kld + (j - 1) * 9 + e]);   // A operand of the blend GEMM
                else pose_map[(size_t)f * Kp + (j - 1) * 9 + e] = pm;
            }
        if (pm_hi && j == 0)     // shape-blend columns (betas) and the zero padding of the GEMM's K axis
            for (int e = Kp; e < Kld; e++) split_f16(e < Kp + NB ? betas[(size_t)f * NB + e - Kp] : 0.f, pm_hi[(size_t)f * Kld + e], pm_lo[(size_t)f * Kld + e]);
    }
    __syncthreads();
    // kinematic chain (smpl_layer.py:119-130), one tree level per round (the reference walks the joints one by one; a
    // joint only reads its parent, so every joint of a level can go at once - same arithmetic, 52 -> ~10 rounds)
    const int my_depth = j < J ? depth[j] : -1;
    for (int lvl = 0; lvl <= max_depth; lvl++) {
        if (my_depth == lvl) {
            const float* R = sR + j * 9;
            float* G = sG + j * 12;
            if (j == 0) {
                for (int r = 0; r < 3; r++) { G[r * 4 + 0] = R[r * 3]; G[r * 4 + 1] = R[r * 3 + 1]; G[r * 4 + 2] = R[r * 3 + 2]; G[r * 4 + 3] = sJ[r]; }
            } else {
                const int p = parents[j];
                const float* Gp = sG + p * 12;
                const float tx = sJ[j * 3] - sJ[p * 3], ty = sJ[j * 3 + 1] - sJ[p * 3 + 1], tz = sJ[j * 3 + 2] - sJ[p * 3 + 2];
                for (int r = 0; r < 3; r++) {
                    const float g0 = Gp[r * 4], g1 = Gp[r * 4 + 1], g2 = Gp[r * 4 + 2], g3 = Gp[r * 4 + 3];
                    G[r * 4 + 0] = g0 * R[0] + g1 * R[3] + g2 * R[6];
                    G[r * 4 + 1] = g0 * R[1] + g1 * R[4] + g2 * R[7];
                    G[r * 4 + 2] = g0 * R[2] + g1 * R[5] + g2 * R[8];
                    G[r * 4 + 3] = g0 * tx + g1 * ty + g2 * tz + g3;
                }
            }
        }
        __syncthreads();
    }
    if (j < J) {
        const float* G = sG + j * 12;
        float* A = Aout + ((size_t)f * J + j) * 12;
        const float jx = sJ[j * 3], jy = sJ[j * 3 + 1], jz = sJ[j * 3 + 2];
        for (int r = 0; r < 3; r++) {
            A[r * 4 + 0] = G[r * 4 + 0]; A[r * 4 + 1] = G[r * 4 + 1]; A[r * 4 + 2] = G[r * 4 + 2];
            A[r * 4 + 3] = G[r * 4 + 3] - (G[r * 4] * jx + G[r * 4 + 1] * jy + G[r * 4 + 2] * jz);
        }
        if (jtr)
            for (int r = 0; r < 3; r++) jtr[((size_t)f * J + j) * 3 + r] = G[r * 4 + 3] + trans[(size_t)f * 3 + r];
    }
}

__global__ void __launch_bounds__(256)
k_lbs_skin(const float* __restrict__ posedirsT, const float* __restrict__ shapedirsT, const float* __restrict__ v_templT,
           const float* __restrict__ weightsT, const float* __restrict__ Ain, const float* __restrict__ pose_map,
           const float* __restrict__ betas, const float* __restrict__ trans, float* __restrict__ verts,
           int F, int V, int J, int NB, int Kp) {
    extern __shared__ __align__(16) float sm[];
    float* s_pm = sm;                  // [Kp][FB]
    float* s_A = s_pm + Kp * FB;       // [FB][J][12]
    float* s_b = s_A + FB * J * 12;    // [NB][FB]
    float* s_t = s_b + NB * FB;        // [FB][3]
    const int f0 = blockIdx.y * FB, tid = threadIdx.x;
    const int nf = min(FB, F - f0);
    for (int i = tid; i < Kp * FB; i += 256) {
        const int k = i / FB, ff = i % FB;
        s_pm[i] = ff < nf ? pose_map[(size_t)(f0 + ff) * Kp + k] : 0.f;
    }
    for (int i = tid; i < FB * J * 12; i += 256) s_A[i] = (i / (J * 12)) < nf ? Ain[(size_t)f0 * J * 12 + i] : 0.f;
    for (int i = tid; i < NB * FB; i += 256) {
        const int b = i / FB, ff = i % FB;
        s_b[i] = ff < nf ? betas[(size_t)(f0 + ff) * NB + b] : 0.f;
    }
    for (int i = tid; i < FB * 3; i += 256) s_t[i] = (i / 3) < nf ? trans[(size_t)f0 * 3 + i] : 0.f;
    __syncthreads();
    const int v = blockIdx.x * 256 + tid;
    if (v >= V) return;

    float acc[3][FB];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float t0 = v_templT[(size_t)c * V + v];
#pragma unroll
        for (int ff = 0; ff < FB; ff++) acc[c][ff] = t0;
    }
    for (int b = 0; b < NB; b++) {
        const float s0 = shapedirsT[((size_t)b * 3 + 0) * V + v], s1 = shapedirsT[((size_t)b * 3 + 1) * V + v],
                    s2 = shapedirsT[((size_t)b * 3 + 2) * V + v];
#pragma unroll
        for (int ff = 0; ff < FB; ff++) {
            const float bb = s_b[b * FB + ff];
            acc[0][ff] = fmaf(s0, bb, acc[0][ff]); acc[1][ff] = fmaf(s1, bb, acc[1][ff]); acc[2][ff] = fmaf(s2, bb, acc[2][ff]);
        }
    }
#pragma unroll 2
    for (int k = 0; k < Kp; k++) {
        const float p0 = __ldg(posedirsT + ((size_t)k * 3 + 0) * V + v), p1 = __ldg(posedirsT + ((size_t)k * 3 + 1) * V + v),
                    p2 = __ldg(posedirsT + ((size_t)k * 3 + 2) * V + v);
        const float4* pm4 = reinterpret_cast<const float4*>(s_pm + k * FB);
#pragma unroll
        for (int q = 0; q < FB / 4; q++) {
            const float4 m = pm4[q];
            acc[0][q * 4 + 0] = fmaf(p0, m.x, acc[0][q * 4 + 0]); acc[1][q * 4 + 0] = fmaf(p1, m.x, acc[1][q * 4 + 0]); acc[2][q * 4 + 0] = fmaf(p2, m.x, acc[2][q * 4 + 0]);
            acc[0][q * 4 + 1] = fmaf(p0, m.y, acc[0][q * 4 + 1]); acc[1][q * 4 + 1] = fmaf(p1, m.y, acc[1][q * 4 + 1]); acc[2][q * 4 + 1] = fmaf(p2, m.y, acc[2][q * 4 + 1]);
            acc[0][q * 4 + 2] = fmaf(p0, m.z, acc[0][q * 4 + 2]); acc[1][q * 4 + 2] = fmaf(p1, m.z, acc[1][q * 4 + 2]); acc[2][q * 4 + 2] = fmaf(p2, m.z, acc[2][q * 4 + 2]);
            acc[0][q * 4 + 3] = fmaf(p0, m.w, acc[0][q * 4 + 3]); acc[1][q * 4 + 3] = fmaf(p1, m.w, acc[1][q * 4 + 3]); acc[2][q * 4 + 3] = fmaf(p2, m.w, acc[2][q * 4 + 3]);
        }
    }
    // skinning, one frame at a time (keeps the 12-entry transform in registers)
    for (int ff = 0; ff < nf; ff++) {
        float Tm[12];
#pragma unroll
        for (int e = 0; e < 12; e++) Tm[e] = 0.f;
        const float4* A4 = reinterpret_cast<const float4*>(s_A + (size_t)ff * J * 12);
        for (int jn = 0; jn < J; jn++) {
            const float w = __ldg(weightsT + (size_t)jn * V + v);
            const float4 a0 = A4[jn * 3], a1 = A4[jn * 3 + 1], a2 = A4[jn * 3 + 2];
            Tm[0] = fmaf(w, a0.x, Tm[0]); Tm[1] = fmaf(w, a0.y, Tm[1]); Tm[2] = fmaf(w, a0.z, Tm[2]); Tm[3] = fmaf(w, a0.w, Tm[3]);
            Tm[4] = fmaf(w, a1.x, Tm[4]); Tm[5] = fmaf(w, a1.y, Tm[5]); Tm[6] = fmaf(w, a1.z, Tm[6]); Tm[7] = fmaf(w, a1.w, Tm[7]);
            Tm[8] = fmaf(w, a2.x, Tm[8]); Tm[9] = fmaf(w, a2.y, Tm[9]); Tm[10] = fmaf(w, a2.z, Tm[10]); Tm[11] = fmaf(w, a2.w, Tm[11]);
        }
        // acc[.][ff] with a runtime ff: select through a small unrolled switch to stay in registers
        float px = 0.f, py = 0.f, pz = 0.f;
#pragma unroll
        for (int q = 0; q < FB; q++)
            if (q == ff) { px = acc[0][q]; py = acc[1][q]; pz = acc[2][q]; }
        float* o = verts + ((size_t)(f0 + ff) * V + v) * 3;
        o[0] = (Tm[0] * px + Tm[1] * py + Tm[2] * pz + Tm[3]) + s_t[ff * 3 + 0];
        o[1] = (Tm[4] * px + Tm[5] * py + Tm[6] * pz + Tm[7]) + s_t[ff * 3 + 1];
        o[2] = (Tm[8] * px + Tm[9] * py + Tm[10] * pz + Tm[11]) + s_t[ff * 3 + 2];
    }
}


// Second half of the tensor-core path.  The pose blend  P vec(R - I)  and the shape blend  S beta  (the 469 multiply-adds per
// vertex coordinate) are ONE split-precision wgmma GEMM  blend[F][3V] = [pose_map | beta][F][469] . (2^8 [P | S])[3V][469]^T
// (gemm_wgmma.cu; fp16 (hi, lo) pairs, fp32 register accumulation; the 2^8 keeps the mm-scale bases well inside the fp16 normal
// range and is undone exactly below; the metre-scale template stays out of the tensor core's truncating accumulation).
// This kernel finishes a vertex: template + blend, skinning matrix from the
// vertex's non-zero bones only (SMPL weights have <= 4 per vertex; ELL list built at init, dense walk as the fallback),
// transform, translation.  Thread = vertex, block = 256 vertices x FS frames; the A matrices of the frame group live in
// shared memory (neighbouring vertices share bones, so the reads are mostly broadcasts); vertices leave through a
// per-warp staging row as 8-byte coalesced stores.
constexpr int FS = 8;
// NZ > 0: every vertex has at most NZ non-zero bones; its ELL list is padded with (bone 0, weight 0), whose products are
// exact zeros, so the loop runs NZ times without a predicate (a predicated-off instruction still costs an issue slot).
// NZ == 0: dense walk over all J bones of weightsT.
template <int NZ>
__global__ void __launch_bounds__(256, 3)
k_lbs_skin_sparse(const float* __restrict__ blend, int ldb, const float* __restrict__ v_templT,
                  const unsigned char* __restrict__ sk_j, const float* __restrict__ sk_w,
                  const float* __restrict__ weightsT, const float* __restrict__ Ain,
                  const float* __restrict__ trans, float* __restrict__ verts, int F, int V, int J) {
    extern __shared__ __align__(16) float sm[];
    float* s_A = sm;                       // [FS][J][12]
    float* s_t = s_A + FS * J * 12;        // [FS][4]
    float* s_o = s_t + FS * 4;             // [8 warps][96] output staging
    const int f0 = blockIdx.y * FS, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nf = min(FS, F - f0);
    const int v0 = blockIdx.x * 256 + warp * 32, v = v0 + lane;
    const int vc = v < V ? v : V - 1;
    // every global read of the thread is issued before its first use: one memory latency per block
    float bl[FS][3];
#pragma unroll
    for (int ff = 0; ff < FS; ff++) {
        const float* q = blend + (size_t)min(f0 + ff, F - 1) * ldb + (size_t)vc * 3;
        bl[ff][0] = q[0]; bl[ff][1] = q[1]; bl[ff][2] = q[2];
    }
    const float vt0 = v_templT[vc], vt1 = v_templT[(size_t)V + vc], vt2 = v_templT[(size_t)2 * V + vc];
    int bj[NZ > 0 ? NZ : 1]; float bw[NZ > 0 ? NZ : 1];
#pragma unroll
    for (int e = 0; e < NZ; e++) { bj[e] = 3 * (int)sk_j[(size_t)e * V + vc]; bw[e] = sk_w[(size_t)e * V + vc]; }
    for (int i = tid; i < nf * J * 12; i += 256) s_A[i] = Ain[(size_t)f0 * J * 12 + i];
    for (int i = tid; i < nf * 3; i += 256) s_t[(i / 3) * 4 + i % 3] = trans[(size_t)f0 * 3 + i];
    __syncthreads();
    float* so = s_o + warp * 96;
    const int nfl = min(32, V - v0) * 3;          // floats of this warp's live vertices (<= 0 for a warp past the end)
#pragma unroll
    for (int ff = 0; ff < FS; ff++) {
        if (ff >= nf) break;
        const float px = fmaf(bl[ff][0], 1.0f / 256.0f, vt0), py = fmaf(bl[ff][1], 1.0f / 256.0f, vt1), pz = fmaf(bl[ff][2], 1.0f / 256.0f, vt2);
        float Tm[12];
#pragma unroll
        for (int e = 0; e < 12; e++) Tm[e] = 0.f;
        const float4* A4 = reinterpret_cast<const float4*>(s_A + (size_t)ff * J * 12);
        if (NZ > 0) {
#pragma unroll
            for (int e = 0; e < NZ; e++) {
                const float w = bw[e];
                const float4 a0 = A4[bj[e]], a1 = A4[bj[e] + 1], a2 = A4[bj[e] + 2];
                Tm[0] = fmaf(w, a0.x, Tm[0]); Tm[1] = fmaf(w, a0.y, Tm[1]); Tm[2] = fmaf(w, a0.z, Tm[2]); Tm[3] = fmaf(w, a0.w, Tm[3]);
                Tm[4] = fmaf(w, a1.x, Tm[4]); Tm[5] = fmaf(w, a1.y, Tm[5]); Tm[6] = fmaf(w, a1.z, Tm[6]); Tm[7] = fmaf(w, a1.w, Tm[7]);
                Tm[8] = fmaf(w, a2.x, Tm[8]); Tm[9] = fmaf(w, a2.y, Tm[9]); Tm[10] = fmaf(w, a2.z, Tm[10]); Tm[11] = fmaf(w, a2.w, Tm[11]);
            }
        } else {
            for (int jn = 0; jn < J; jn++) {
                const float w = __ldg(weightsT + (size_t)jn * V + vc);
                const float4 a0 = A4[jn * 3], a1 = A4[jn * 3 + 1], a2 = A4[jn * 3 + 2];
                Tm[0] = fmaf(w, a0.x, Tm[0]); Tm[1] = fmaf(w, a0.y, Tm[1]); Tm[2] = fmaf(w, a0.z, Tm[2]); Tm[3] = fmaf(w, a0.w, Tm[3]);
                Tm[4] = fmaf(w, a1.x, Tm[4]); Tm[5] = fmaf(w, a1.y, Tm[5]); Tm[6] = fmaf(w, a1.z, Tm[6]); Tm[7] = fmaf(w, a1.w, Tm[7]);
                Tm[8] = fmaf(w, a2.x, Tm[8]); Tm[9] = fmaf(w, a2.y, Tm[9]); Tm[10] = fmaf(w, a2.z, Tm[10]); Tm[11] = fmaf(w, a2.w, Tm[11]);
            }
        }
        so[lane * 3 + 0] = (Tm[0] * px + Tm[1] * py + Tm[2] * pz + Tm[3]) + s_t[ff * 4 + 0];
        so[lane * 3 + 1] = (Tm[4] * px + Tm[5] * py + Tm[6] * pz + Tm[7]) + s_t[ff * 4 + 1];
        so[lane * 3 + 2] = (Tm[8] * px + Tm[9] * py + Tm[10] * pz + Tm[11]) + s_t[ff * 4 + 2];
        __syncwarp();
        // 96 floats of this warp's 32 vertices are contiguous in verts[f][v0 .. v0+31][3]
        float* dst = verts + ((size_t)(f0 + ff) * V + v0) * 3;
        if (nfl == 96 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
            *reinterpret_cast<float2*>(dst + lane * 2) = *reinterpret_cast<const float2*>(so + lane * 2);
            if (lane < 16) *reinterpret_cast<float2*>(dst + 64 + lane * 2) = *reinterpret_cast<const float2*>(so + 64 + lane * 2);
        } else {
            for (int i = lane; i < nfl; i += 32) dst[i] = so[i];
        }
        __syncwarp();
    }
}

}  // namespace

void idb_body_release(idb_handle* h) {
    if (!h->body) return;
    h->epoch++;
    BodyModel& m = *h->body;
    for (void* p : m.owned) cudaFree(p);
    if (m.A) { cudaFree(m.A); cudaFree(m.pose_map); cudaFree(m.pm_hi); cudaFree(m.blend); }
    delete h->body;
    h->body = nullptr;
}

extern "C" int idb_body_init(idb_handle* h, int V, int J, int NB, int Fc, const float* v_template, const float* shapedirs,
                             const float* posedirs, const float* J_regressor, const float* weights,
                             const int32_t* parents, const int32_t* faces) {
    IDB_ENTER(h);
    if (!h || !v_template || !shapedirs || !posedirs || !J_regressor || !weights || !parents) return IDB_ERR_ARG;
    if (V <= 0 || J <= 1 || J > 64 || NB <= 0 || NB > 16) return idb_fail(h, IDB_ERR_ARG, "bad body model dimensions");
    idb_body_release(h);
    h->body = new BodyModel();
    BodyModel& m = *h->body;
    m.V = V; m.J = J; m.NB = NB; m.Fc = Fc; m.Kp = (J - 1) * 9;
    const int Kp = m.Kp;
    auto pull = [&](const void* src, size_t bytes, void* dst) { return cudaMemcpy(dst, src, bytes, cudaMemcpyDefault); };
    std::vector<float> vt((size_t)V * 3), sd((size_t)V * 3 * NB), pd((size_t)V * 3 * Kp), jr((size_t)J * V), w((size_t)V * J);
    std::vector<int32_t> par(J);
    CUDA_TRY(h, pull(v_template, vt.size() * 4, vt.data())); CUDA_TRY(h, pull(shapedirs, sd.size() * 4, sd.data()));
    CUDA_TRY(h, pull(posedirs, pd.size() * 4, pd.data())); CUDA_TRY(h, pull(J_regressor, jr.size() * 4, jr.data()));
    CUDA_TRY(h, pull(weights, w.size() * 4, w.data())); CUDA_TRY(h, pull(parents, par.size() * 4, par.data()));
    for (int i = 1; i < J; i++)
        if (par[i] < 0 || par[i] >= i) return idb_fail(h, IDB_ERR_ARG, "parents must precede children (joint %d)", i);
    std::vector<float> vtT((size_t)3 * V), sdT((size_t)NB * 3 * V), pdT((size_t)Kp * 3 * V), wT((size_t)J * V);
    for (int v = 0; v < V; v++)
        for (int c = 0; c < 3; c++) {
            vtT[(size_t)c * V + v] = vt[(size_t)v * 3 + c];
            for (int b = 0; b < NB; b++) sdT[((size_t)b * 3 + c) * V + v] = sd[((size_t)v * 3 + c) * NB + b];
            for (int k = 0; k < Kp; k++) pdT[((size_t)k * 3 + c) * V + v] = pd[((size_t)v * 3 + c) * Kp + k];
        }
    for (int v = 0; v < V; v++) for (int j = 0; j < J; j++) wT[(size_t)j * V + v] = w[(size_t)v * J + j];
    std::vector<float> Jt((size_t)J * 3), Js((size_t)J * 3 * NB);
    for (int j = 0; j < J; j++)
        for (int c = 0; c < 3; c++) {
            double a = 0;
            for (int v = 0; v < V; v++) a += (double)jr[(size_t)j * V + v] * vt[(size_t)v * 3 + c];
            Jt[j * 3 + c] = (float)a;
            for (int b = 0; b < NB; b++) {
                double s = 0;
                for (int v = 0; v < V; v++) s += (double)jr[(size_t)j * V + v] * sd[((size_t)v * 3 + c) * NB + b];
                Js[((size_t)j * 3 + c) * NB + b] = (float)s;
            }
        }
    auto up = [&](const void* src, size_t bytes, void** dst) {
        cudaError_t e = cudaMalloc(dst, bytes ? bytes : 4);
        if (e == cudaSuccess) e = cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) m.owned.push_back(*dst);
        return e;
    };
    CUDA_TRY(h, up(vtT.data(), vtT.size() * 4, (void**)&m.v_templT)); CUDA_TRY(h, up(sdT.data(), sdT.size() * 4, (void**)&m.shapedirsT));
    CUDA_TRY(h, up(pdT.data(), pdT.size() * 4, (void**)&m.posedirsT)); CUDA_TRY(h, up(wT.data(), wT.size() * 4, (void**)&m.weightsT));
    CUDA_TRY(h, up(Jt.data(), Jt.size() * 4, (void**)&m.J_templ)); CUDA_TRY(h, up(Js.data(), Js.size() * 4, (void**)&m.J_shape));
    CUDA_TRY(h, up(par.data(), par.size() * 4, (void**)&m.parents));
    {
        std::vector<int32_t> dep(J, 0);
        for (int i = 1; i < J; i++) { dep[i] = dep[par[i]] + 1; if (dep[i] > m.max_depth) m.max_depth = dep[i]; }
        CUDA_TRY(h, up(dep.data(), dep.size() * 4, (void**)&m.depth));
    }
    {
        // tensor-core pose blend: W operand of the GEMM = 2^8 * posedirs in its native (V,3,Kp) order (row n = v*3 + c)
        // K axis of the GEMM = [459 pose-blend terms | NB shape-blend terms]: both are cm-scale corrections of the template
        const int Kb = Kp + NB;
        m.Nb = (3 * V + 255) & ~255; m.Kld = (Kb + 7) & ~7;     // whole 256-column GEMM tiles
        std::vector<float> pds((size_t)m.Nb * Kb, 0.f);
        for (size_t n = 0; n < (size_t)3 * V; n++) {
            for (int k = 0; k < Kp; k++) pds[n * Kb + k] = pd[n * Kp + k] * 256.0f;
            for (int b = 0; b < NB; b++) pds[n * Kb + Kp + b] = sd[n * NB + b] * 256.0f;
        }
        float* tmp = nullptr;
        CUDA_TRY(h, cudaMalloc((void**)&tmp, pds.size() * 4));
        cudaError_t e = cudaMemcpy(tmp, pds.data(), pds.size() * 4, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMalloc((void**)&m.pd_hi, (size_t)m.Nb * m.Kld * sizeof(__half) * 2 + 64);
        if (e != cudaSuccess) { cudaFree(tmp); return idb_fail(h, IDB_ERR_CUDA, "posedirs pairs: %s", cudaGetErrorString(e)); }
        m.owned.push_back(m.pd_hi);
        m.pd_lo = m.pd_hi + (size_t)m.Nb * m.Kld;
        int rc = idb_split_tensor(h, tmp, Kb, m.pd_hi, m.pd_lo, m.Kld, m.Nb, Kb, 0);
        cudaDeviceSynchronize();
        cudaFree(tmp);
        if (rc) return rc;
        // skinning weights: non-zero bones per vertex (ELL, bone-major so a warp reads consecutive vertices)
        std::vector<unsigned char> skn(V, 0), skj((size_t)SK_MAX * V, 0);
        std::vector<float> skw((size_t)SK_MAX * V, 0.f);
        m.sk_dense = false;
        for (int v = 0; v < V && !m.sk_dense; v++) {
            int n = 0;
            for (int j = 0; j < J; j++)
                if (w[(size_t)v * J + j] != 0.f) {
                    if (n == SK_MAX) { m.sk_dense = true; break; }
                    skj[(size_t)n * V + v] = (unsigned char)j; skw[(size_t)n * V + v] = w[(size_t)v * J + j]; n++;
                }
            skn[v] = (unsigned char)n;
            if (n > m.sk_max) m.sk_max = n;
        }
        CUDA_TRY(h, up(skn.data(), skn.size(), (void**)&m.sk_n)); CUDA_TRY(h, up(skj.data(), skj.size(), (void**)&m.sk_j));
        CUDA_TRY(h, up(skw.data(), skw.size() * 4, (void**)&m.sk_w));
    }
    if (faces && Fc > 0) {
        std::vector<int32_t> fc((size_t)Fc * 3);
        CUDA_TRY(h, pull(faces, fc.size() * 4, fc.data()));
        // vertex -> incident (face, corner) list in the reference's accumulation order
        // (data/tools.py:26-34: all corner-1 adds, then corner-2, then corner-0; index_add_ is
        // sequential in face order on CPU)
        std::vector<int32_t> off(V + 1, 0), ent;
        const int order[3] = {1, 2, 0};
        for (int pass = 0; pass < 3; pass++)
            for (int f = 0; f < Fc; f++) {
                int vv = fc[(size_t)f * 3 + order[pass]];
                if (vv < 0 || vv >= V) return idb_fail(h, IDB_ERR_ARG, "face index out of range");
                off[vv + 1]++;
            }
        for (int v = 0; v < V; v++) off[v + 1] += off[v];
        ent.resize((size_t)Fc * 3);
        std::vector<int32_t> cur(off.begin(), off.end() - 1);
        for (int pass = 0; pass < 3; pass++)
            for (int f = 0; f < Fc; f++) {
                int vv = fc[(size_t)f * 3 + order[pass]];
                ent[cur[vv]++] = f * 4 + order[pass];
            }
        CUDA_TRY(h, up(fc.data(), fc.size() * 4, (void**)&m.faces));
        CUDA_TRY(h, up(off.data(), off.size() * 4, (void**)&m.vf_off));
        CUDA_TRY(h, up(ent.data(), ent.size() * 4, (void**)&m.vf_ent));
    }
    // Vertex clusters for the pruned nearest-neighbour search (geometry.cu): k-means on the template; clusters of
    // neighbouring template vertices stay compact under articulation.  Any partition is CORRECT (bounds are
    // recomputed from the posed vertices of every frame); compactness only decides how much gets pruned.
    if (V <= 65535) {
        const int C = NN_CLUSTERS;
        std::vector<double> cx(C), cy(C), cz(C);
        for (int c = 0; c < C; c++) {
            const int v = (int)((long long)c * V / C);
            cx[c] = vt[(size_t)v * 3]; cy[c] = vt[(size_t)v * 3 + 1]; cz[c] = vt[(size_t)v * 3 + 2];
        }
        std::vector<int> asg(V, 0);
        for (int it = 0; it < 10; it++) {
            for (int v = 0; v < V; v++) {
                double best = 1e300; int bc = 0;
                for (int c = 0; c < C; c++) {
                    const double dx = vt[(size_t)v * 3] - cx[c], dy = vt[(size_t)v * 3 + 1] - cy[c], dz = vt[(size_t)v * 3 + 2] - cz[c];
                    const double d = dx * dx + dy * dy + dz * dz;
                    if (d < best) { best = d; bc = c; }
                }
                asg[v] = bc;
            }
            std::vector<double> sx(C, 0), sy(C, 0), sz(C, 0); std::vector<int> cnt(C, 0);
            for (int v = 0; v < V; v++) { const int c = asg[v]; sx[c] += vt[(size_t)v * 3]; sy[c] += vt[(size_t)v * 3 + 1]; sz[c] += vt[(size_t)v * 3 + 2]; cnt[c]++; }
            for (int c = 0; c < C; c++) if (cnt[c]) { cx[c] = sx[c] / cnt[c]; cy[c] = sy[c] / cnt[c]; cz[c] = sz[c] / cnt[c]; }
        }
        std::vector<int32_t> off(C + 1, 0);
        for (int v = 0; v < V; v++) off[asg[v] + 1]++;
        for (int c = 0; c < C; c++) off[c + 1] += off[c];
        std::vector<uint16_t> vid(V);
        std::vector<int32_t> cur(off.begin(), off.end() - 1);
        for (int v = 0; v < V; v++) vid[cur[asg[v]]++] = (uint16_t)v;      // ascending ids inside a cluster
        CUDA_TRY(h, up(vid.data(), vid.size() * sizeof(uint16_t), (void**)&m.nn_vid));
        CUDA_TRY(h, up(off.data(), off.size() * 4, (void**)&m.nn_off));
    }
    // the opt-in is a per-function, per-device limit (NOT per model): always raise it to the device maximum, or a second,
    // smaller body model on the same device would lower it under the first one's launches
    const int smem_skin = (int)sizeof(float) * (Kp * FB + FB * J * 12 + NB * FB + FB * 3);
    if (smem_skin > 227 * 1024) return idb_fail(h, IDB_ERR_ARG, "body model too large for the SIMT skinning kernel's shared memory");
    CUDA_TRY(h, cudaFuncSetAttribute(k_lbs_skin, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CUDA_TRY(h, cudaFuncSetAttribute(k_lbs_skin_sparse<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CUDA_TRY(h, cudaFuncSetAttribute(k_lbs_skin_sparse<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CUDA_TRY(h, cudaFuncSetAttribute(k_lbs_skin_sparse<SK_MAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    h->epoch++;
    return IDB_OK;
}

int idb_body_workspace(idb_handle* h, int F) {
    BodyModel& m = *h->body;
    if (F <= m.capF) return IDB_OK;
    h->epoch++;                      // captured loop graphs point at the old workspace
    if (m.A) { cudaFree(m.A); cudaFree(m.pose_map); cudaFree(m.pm_hi); cudaFree(m.blend); }
    m.A = nullptr; m.capF = 0;
    CUDA_TRY(h, cudaMalloc((void**)&m.A, sizeof(float) * (size_t)F * m.J * 12));
    CUDA_TRY(h, cudaMalloc((void**)&m.pose_map, sizeof(float) * (size_t)F * m.Kp));
    CUDA_TRY(h, cudaMalloc((void**)&m.pm_hi, sizeof(__half) * 2 * (size_t)F * m.Kld + 64));
    CUDA_TRY(h, cudaMalloc((void**)&m.blend, sizeof(float) * (size_t)F * m.Nb));
    m.pm_lo = m.pm_hi + (size_t)F * m.Kld;
    m.capF = F;
    return IDB_OK;
}

extern "C" int idb_smplh_lbs(idb_handle* h, int F, const float* pose, const float* betas, const float* trans,
                             float* verts, float* jtr, void* stream) {
    IDB_ENTER(h);
    if (!h || !pose || !betas || !trans || F <= 0) return IDB_ERR_ARG;
    if (!h->body) return idb_fail(h, IDB_ERR_STATE, "idb_body_init first");
    BodyModel& m = *h->body;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = idb_body_workspace(h, F);
    if (rc) return rc;
    const size_t smem_pose = sizeof(float) * (size_t)m.J * (9 + 3 + 12);
    // tensor backend: the 459-term pose blend is a split-precision wgmma GEMM, the rest a sparse-bone skinning kernel
    const bool tensor = h->gemm_backend == 1 && verts && m.pd_hi;
    k_lbs_pose<<<F, 64, smem_pose, st>>>(pose, betas, trans, m.J_templ, m.J_shape, m.parents, m.A, m.pose_map, jtr, m.J, m.NB, m.Kp,
                                         tensor ? m.pm_hi : nullptr, tensor ? m.pm_lo : nullptr, m.Kld, m.depth, m.max_depth);
    LAUNCH_CHECK(h);
    if (tensor) {
        GemmArgs g;
        g.A_hi = m.pm_hi; g.A_lo = m.pm_lo; g.lda = m.Kld; g.W_hi = m.pd_hi; g.W_lo = m.pd_lo; g.ldw = m.Kld;
        g.C = m.blend; g.ldc = m.Nb; g.M = F; g.N = m.Nb; g.K = m.Kld; g.epi = 0; g.single_acc = 1;
        if ((rc = idb_gemm_ex(h, g, st))) return rc;
        const size_t smem = sizeof(float) * ((size_t)FS * m.J * 12 + FS * 4 + 8 * 96);
        dim3 grid((m.V + 255) / 256, (F + FS - 1) / FS);
        if (m.sk_dense)
            k_lbs_skin_sparse<0><<<grid, 256, smem, st>>>(m.blend, m.Nb, m.v_templT, m.sk_j, m.sk_w, m.weightsT, m.A, trans, verts, F, m.V, m.J);
        else if (m.sk_max <= 4)
            k_lbs_skin_sparse<4><<<grid, 256, smem, st>>>(m.blend, m.Nb, m.v_templT, m.sk_j, m.sk_w, m.weightsT, m.A, trans, verts, F, m.V, m.J);
        else
            k_lbs_skin_sparse<SK_MAX><<<grid, 256, smem, st>>>(m.blend, m.Nb, m.v_templT, m.sk_j, m.sk_w, m.weightsT, m.A, trans, verts, F, m.V, m.J);
        LAUNCH_CHECK(h);
    } else if (verts) {
        const size_t smem_skin = sizeof(float) * ((size_t)m.Kp * FB + (size_t)FB * m.J * 12 + (size_t)m.NB * FB + FB * 3);
        dim3 grid((m.V + 255) / 256, (F + FB - 1) / FB);
        k_lbs_skin<<<grid, 256, smem_skin, st>>>(m.posedirsT, m.shapedirsT, m.v_templT, m.weightsT, m.A, m.pose_map, betas, trans,
                                                  verts, F, m.V, m.J, m.NB, m.Kp);
        LAUNCH_CHECK(h);
    }
    return IDB_OK;
}
