// Geometry helpers around the loop (fp32).
//   vertex normals      : reference data/tools.py:4-39
//   signed nearest point: reference tools.py:11-76 (+ the chamfer_distance CUDA ext it calls,
//                         tools.py:45-47: first-minimum squared-L2 argmin)
//   rot6d -> axis-angle : pytorch3d.transforms 0.7.2 rotation_6d_to_matrix / matrix_to_quaternion
//                         / quaternion_to_axis_angle (reference eval_smpl_short.py:90-91,157-162)
#include "common.cuh"
#include "body.cuh"
#include "rot.cuh"

namespace {

// One thread per (frame, vertex); gathers the incident faces in the reference's accumulation
// order (no atomics => deterministic).
__global__ void k_vertex_normals(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                 const int32_t* __restrict__ vf_off, const int32_t* __restrict__ vf_ent,
                                 float* __restrict__ normals, int V) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = blockIdx.y;
    if (v >= V) return;
    const float* vb = verts + (size_t)f * V * 3;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (int e = vf_off[v]; e < vf_off[v + 1]; e++) {
        const int ent = vf_ent[e], fi = ent >> 2, corner = ent & 3;
        const int i0 = faces[fi * 3], i1 = faces[fi * 3 + 1], i2 = faces[fi * 3 + 2];
        // corner 1: (v2-v1)x(v0-v1); corner 2: (v0-v2)x(v1-v2); corner 0: (v1-v0)x(v2-v0)
        const int ic = corner == 0 ? i0 : (corner == 1 ? i1 : i2);
        const int ia = corner == 0 ? i1 : (corner == 1 ? i2 : i0);
        const int ib = corner == 0 ? i2 : (corner == 1 ? i0 : i1);
        const float cx = vb[ic * 3], cy = vb[ic * 3 + 1], cz = vb[ic * 3 + 2];
        const float ax = vb[ia * 3] - cx, ay = vb[ia * 3 + 1] - cy, az = vb[ia * 3 + 2] - cz;
        const float bx = vb[ib * 3] - cx, by = vb[ib * 3 + 1] - cy, bz = vb[ib * 3 + 2] - cz;
        nx += ay * bz - az * by;
        ny += az * bx - ax * bz;
        nz += ax * by - ay * bx;
    }
    const float len = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-6f);  // F.normalize(eps=1e-6)
    float* o = normals + ((size_t)f * V + v) * 3;
    o[0] = nx / len; o[1] = ny / len; o[2] = nz / len;
}

// Brute-force nearest target per query, one frame per blockIdx.y, 256 queries per block, targets
// staged through shared memory in tiles.  d = (dx*dx + dy*dy) + dz*dz without FMA contraction and
// strict '<' so the FIRST minimum wins (same as the restated argmin in oracle/restate.py).
constexpr int NN_TILE = 1024;
__global__ void __launch_bounds__(256)
k_signed_nn(const float* __restrict__ query, const float* __restrict__ target, const float* __restrict__ tnormals,
            float* __restrict__ sdist, int32_t* __restrict__ idx_out, float* __restrict__ vec_out, int Pq, int Pt) {
    __shared__ float4 st[NN_TILE];
    const int f = blockIdx.y, q = blockIdx.x * 256 + threadIdx.x;
    const float* qb = query + (size_t)f * Pq * 3;
    const float* tb = target + (size_t)f * Pt * 3;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (q < Pq) { qx = qb[q * 3]; qy = qb[q * 3 + 1]; qz = qb[q * 3 + 2]; }
    float best = INFINITY;
    int bi = 0;
    for (int t0 = 0; t0 < Pt; t0 += NN_TILE) {
        const int nt = min(NN_TILE, Pt - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < nt; i += 256)
            st[i] = make_float4(tb[(size_t)(t0 + i) * 3], tb[(size_t)(t0 + i) * 3 + 1], tb[(size_t)(t0 + i) * 3 + 2], 0.f);
        __syncthreads();
#pragma unroll 4
        for (int i = 0; i < nt; i++) {
            const float4 t = st[i];
            const float dx = qx - t.x, dy = qy - t.y, dz = qz - t.z;
            const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            if (d < best) { best = d; bi = t0 + i; }
        }
    }
    if (q >= Pq) return;
    const float vx = qx - tb[(size_t)bi * 3], vy = qy - tb[(size_t)bi * 3 + 1], vz = qz - tb[(size_t)bi * 3 + 2];
    float d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz)));
    if (tnormals) {
        const float* n = tnormals + ((size_t)f * Pt + bi) * 3;
        const float dot = __fadd_rn(__fadd_rn(__fmul_rn(n[0], vx), __fmul_rn(n[1], vy)), __fmul_rn(n[2], vz));
        d *= (dot > 0.f) ? 1.0f : ((dot < 0.f) ? -1.0f : 0.0f);
    }
    const size_t o = (size_t)f * Pq + q;
    if (sdist) sdist[o] = d;
    if (idx_out) idx_out[o] = bi;
    if (vec_out) { vec_out[o * 3] = vx; vec_out[o * 3 + 1] = vy; vec_out[o * 3 + 2] = vz; }
}

// Same result as k_signed_nn, bit for bit, with most of the 6890 candidates pruned.  The target vertices come
// grouped into NN_CLUSTERS clusters (BodyModel::nn_vid / nn_off).  One block = one frame x a chunk of queries:
// it stages the frame's vertices cluster-sorted in shared memory and computes an axis-aligned bounding box per cluster
// from the POSED vertices; then one warp per query: box distances for 8 clusters per lane, a seed scan of the nearest box, and
// a walk over the boxes within the seed bound that re-tests each against the current best distance.  Candidate
// distances use exactly the brute-force expression, candidates compare lexicographically on (distance, vertex
// id), and a cluster holding a vertex at the final minimum distance can never be skipped (that distance is <= d0),
// so the FIRST minimum of the brute-force scan is reproduced.
__device__ __forceinline__ float nn_dist2(float qx, float qy, float qz, float x, float y, float z) {
    const float dx = qx - x, dy = qy - y, dz = qz - z;
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__global__ void __launch_bounds__(512)
k_signed_nn_pruned(const float* __restrict__ query, const float* __restrict__ target, const float* __restrict__ tnormals,
                   float* __restrict__ sdist, int32_t* __restrict__ idx_out, float* __restrict__ vec_out, int Pq, int Pt,
                   const uint16_t* __restrict__ vid_sorted, const int32_t* __restrict__ coff, int qchunk) {
    extern __shared__ __align__(16) float nsm[];
    const int Ptp = (Pt + 3) & ~3;
    float* xs = nsm; float* ys = xs + Ptp; float* zs = ys + Ptp;
    float4* cen = reinterpret_cast<float4*>(zs + Ptp);                 // box centre xyz, w < 0: empty cluster
    float4* ext = cen + NN_CLUSTERS;                                    // box half extents (slightly inflated)
    int32_t* off = reinterpret_cast<int32_t*>(ext + NN_CLUSTERS);       // [NN_CLUSTERS + 1] (+3 pad)
    uint16_t* vid = reinterpret_cast<uint16_t*>(off + NN_CLUSTERS + 4);
    const int f = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* qb = query + (size_t)f * Pq * 3;
    const float* tb = target + (size_t)f * Pt * 3;
    for (int i = tid; i < Pt; i += 512) {
        const int v = vid_sorted[i];
        vid[i] = (uint16_t)v;
        xs[i] = tb[(size_t)v * 3]; ys[i] = tb[(size_t)v * 3 + 1]; zs[i] = tb[(size_t)v * 3 + 2];
    }
    for (int i = tid; i <= NN_CLUSTERS; i += 512) off[i] = coff[i];
    __syncthreads();
    for (int c = tid; c < NN_CLUSTERS; c += 512) {
        const int b = off[c], e = off[c + 1];
        // axis-aligned bounding box of the cluster's POSED vertices (patches of a body surface are flat: a box bounds them
        // far more tightly than a sphere); half extents inflated so that centre +- extent covers min / max despite rounding
        float4 o = make_float4(0.f, 0.f, 0.f, -1.f), hx = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e > b) {
            float lx = xs[b], ly = ys[b], lz = zs[b], ux = lx, uy = ly, uz = lz;
            for (int i = b + 1; i < e; i++) {
                lx = fminf(lx, xs[i]); ly = fminf(ly, ys[i]); lz = fminf(lz, zs[i]);
                ux = fmaxf(ux, xs[i]); uy = fmaxf(uy, ys[i]); uz = fmaxf(uz, zs[i]);
            }
            o = make_float4(0.5f * (lx + ux), 0.5f * (ly + uy), 0.5f * (lz + uz), 1.f);
            hx = make_float4(0.5f * (ux - lx) * 1.00001f + 1e-6f * (1.0f + fabsf(o.x)), 0.5f * (uy - ly) * 1.00001f + 1e-6f * (1.0f + fabsf(o.y)),
                             0.5f * (uz - lz) * 1.00001f + 1e-6f * (1.0f + fabsf(o.z)), 0.f);
        }
        cen[c] = o; ext[c] = hx;
    }
    __syncthreads();
    const int q0 = blockIdx.x * qchunk, q1 = min(Pq, q0 + qchunk);
    for (int q = q0 + warp; q < q1; q += 16) {
        const float qx = qb[q * 3], qy = qb[q * 3 + 1], qz = qb[q * 3 + 2];
        // clusters lane + 32k: lower bound lb2 of the squared distance to any vertex of the cluster (distance to its box;
        // empty clusters: +inf).  (1) seed: the cluster with the (approximately) smallest lower bound - one redux on a packed
        // (distance bits | cluster id) key - is scanned first; (2) candidate mask: clusters whose box is within the seed
        // bound (2e-4 relative slack on the safe side, inclusive so that ties are visited); (3) the candidates are walked in
        // id order, each re-tested against the CURRENT warp-uniform bound (one shuffle for its lower bound, one redux.min on
        // the distance bits after every scan), so clusters that stopped mattering are skipped for 4 instructions.  (A strict
        // best-first order costs a per-step arg-min that outweighs the scans it saves.)
        float lb2[NN_CLUSTERS / 32];
        unsigned key = 0xffffffffu;
#pragma unroll
        for (int k = 0; k < NN_CLUSTERS / 32; k++) {
            const int c = lane + 32 * k;
            const float4 cc = cen[c], hh = ext[c];
            const float ex = fmaxf(fabsf(qx - cc.x) - hh.x, 0.f), ey = fmaxf(fabsf(qy - cc.y) - hh.y, 0.f), ez = fmaxf(fabsf(qz - cc.z) - hh.z, 0.f);
            lb2[k] = cc.w >= 0.f ? (ex * ex + ey * ey) + ez * ez : INFINITY;
            key = min(key, (__float_as_uint(lb2[k]) & 0xffffff00u) | (unsigned)c);      // non-negative floats order like their bit patterns
        }
        const int cmin = (int)(__reduce_min_sync(0xffffffffu, key) & 0xffu);
        float bd = INFINITY; int bi = 0x7fffffff;
        {
            const int b = off[cmin], e = off[cmin + 1];
            for (int i = b + lane; i < e; i += 32) {
                const float d = nn_dist2(qx, qy, qz, xs[i], ys[i], zs[i]);
                const int v = vid[i];
                if (d < bd || (d == bd && v < bi)) { bd = d; bi = v; }
            }
        }
        // warp-uniform bound = smallest candidate distance so far (bit pattern of a non-negative float; +inf when none / NaN)
        unsigned bound_u = __reduce_min_sync(0xffffffffu, bd == bd ? __float_as_uint(bd) : 0x7f800000u);
#pragma unroll
        for (int k = 0; k < NN_CLUSTERS / 32; k++) {
            const float lbk = lb2[k];
            unsigned m = __ballot_sync(0xffffffffu, lbk * 0.9999f <= __uint_as_float(bound_u) * 1.0002f && (lane + 32 * k) != cmin);
            while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                const float lbc = __shfl_sync(0xffffffffu, lbk, src);
                if (!(lbc * 0.9999f <= __uint_as_float(bound_u) * 1.0002f)) continue;          // the bound moved since the mask was taken
                const int c = src + 32 * k;
                const int b = off[c], e = off[c + 1];
                for (int i = b + lane; i < e; i += 32) {
                    const float d = nn_dist2(qx, qy, qz, xs[i], ys[i], zs[i]);
                    const int v = vid[i];
                    if (d < bd || (d == bd && v < bi)) { bd = d; bi = v; }
                }
                bound_u = min(bound_u, __reduce_min_sync(0xffffffffu, bd == bd ? __float_as_uint(bd) : 0x7f800000u));
            }
        }
        __syncwarp();
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const float od = __shfl_xor_sync(0xffffffffu, bd, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
        }
        if (lane == 0) {
            if (bi == 0x7fffffff) bi = 0;      // no finite distance (NaN input): same answer as the brute-force scan
            const float vx = qx - tb[(size_t)bi * 3], vy = qy - tb[(size_t)bi * 3 + 1], vz = qz - tb[(size_t)bi * 3 + 2];
            float d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz)));
            if (tnormals) {
                const float* n = tnormals + ((size_t)f * Pt + bi) * 3;
                const float dot = __fadd_rn(__fadd_rn(__fmul_rn(n[0], vx), __fmul_rn(n[1], vy)), __fmul_rn(n[2], vz));
                d *= (dot > 0.f) ? 1.0f : ((dot < 0.f) ? -1.0f : 0.0f);
            }
            const size_t o = (size_t)f * Pq + q;
            if (sdist) sdist[o] = d;
            if (idx_out) idx_out[o] = bi;
            if (vec_out) { vec_out[o * 3] = vx; vec_out[o * 3 + 1] = vy; vec_out[o * 3 + 2] = vz; }
        }
    }
}

}  // namespace

namespace {
__global__ void k_rot6d_to_aa(const float* __restrict__ d6, float* __restrict__ aa, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float in[6], R[9], o[3];
    for (int k = 0; k < 6; k++) in[k] = d6[(size_t)i * 6 + k];
    idb_rot6d_to_matrix(in, R);
    idb_matrix_to_axis_angle(R, o);
    aa[(size_t)i * 3] = o[0]; aa[(size_t)i * 3 + 1] = o[1]; aa[(size_t)i * 3 + 2] = o[2];
}
}  // namespace

extern "C" int idb_vertex_normals(idb_handle* h, int F, const float* verts, float* normals, void* stream) {
    IDB_ENTER(h);
    if (!h || !verts || !normals || F <= 0) return IDB_ERR_ARG;
    if (!h->body || !h->body->faces) return idb_fail(h, IDB_ERR_STATE, "idb_body_init with faces first");
    BodyModel& m = *h->body;
    dim3 grid((m.V + 127) / 128, F);
    k_vertex_normals<<<grid, 128, 0, (cudaStream_t)stream>>>(verts, m.faces, m.vf_off, m.vf_ent, normals, m.V);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

extern "C" int idb_signed_nn(idb_handle* h, int F, int Pq, int Pt, const float* query, const float* target,
                             const float* target_normals, float* signed_dist, int32_t* idx, float* vec, void* stream) {
    IDB_ENTER(h);
    if (!h || !query || !target || F <= 0 || Pq <= 0 || Pt <= 0) return IDB_ERR_ARG;
    // body-mesh targets take the cluster-pruned search (identical results, ~8x fewer candidate evaluations)
    if (h->nn_pruning && h->body && h->body->nn_vid && Pt == h->body->V && Pt <= 12000) {
        const int Ptp = (Pt + 3) & ~3;
        const size_t smem = sizeof(float) * 3 * Ptp + 2 * sizeof(float4) * NN_CLUSTERS + sizeof(int32_t) * (NN_CLUSTERS + 4) + sizeof(uint16_t) * Ptp + sizeof(unsigned) * 16 * (NN_CLUSTERS / 32);
        if (!(h->attr_mask & 4u)) {
            CUDA_TRY(h, cudaFuncSetAttribute(k_signed_nn_pruned, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            h->attr_mask |= 4u;
        }
        const int qchunk = 1024;
        dim3 grid((Pq + qchunk - 1) / qchunk, F);
        k_signed_nn_pruned<<<grid, 512, smem, (cudaStream_t)stream>>>(query, target, target_normals, signed_dist, idx, vec, Pq, Pt,
                                                                      h->body->nn_vid, h->body->nn_off, qchunk);
        LAUNCH_CHECK(h);
        return IDB_OK;
    }
    dim3 grid((Pq + 255) / 256, F);
    k_signed_nn<<<grid, 256, 0, (cudaStream_t)stream>>>(query, target, target_normals, signed_dist, idx, vec, Pq, Pt);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

extern "C" int idb_rot6d_to_axis_angle(idb_handle* h, int n, const float* rot6d, float* aa, void* stream) {
    IDB_ENTER(h);
    if (!h || !rot6d || !aa || n <= 0) return IDB_ERR_ARG;
    k_rot6d_to_aa<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(rot6d, aa, n);
    LAUNCH_CHECK(h);
    return IDB_OK;
}
