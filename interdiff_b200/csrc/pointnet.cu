// PointNet++ (MSG) point-cloud encoder of the conditioning path: MDM.pcEmbedding =
// PointNet2Encoder(c_in=1, c_out=256, num_keypoints=1) (reference model/layers.py:111-175, called from
// model/diffusion_smpl.py:210-211).  SURVEY 8f rank 1, first half.
//
// The reference delegates the point operators to the un-vendored CUDA extension pointnet2_ops 3.0.0
// (furthest_point_sampling, ball_query, group_points; generic SIMT code whose arch list stops at sm_75).
// They are rebuilt here for sm_90a following that version's published algorithm - the same statement the
// oracle (oracle/pointnet2_restated.py) follows, with the same evaluation order of the float32 distances
// ((dx*dx + dy*dy) + dz*dz, no FMA contraction) so that every discrete decision (which point is the
// furthest, which points are in the ball) is reproduced exactly:
//   k_fps      one block per cloud, 512 threads own points t, t+512, ...; per sampled point: min-distance
//              update in registers, thread-best = first point of the walk with the largest value, block
//              reduction = larger value, ties to the lower thread; points with |p|^2 <= 1e-3 are skipped.
//   k_sa1      set abstraction 1 (npoint 1024; radii .05/.1; 16/32 samples): one warp per centre and scale:
//              ballot scan of the cloud in index order (first nsample hits, padded with the first), then the
//              3-layer 1x1-conv MLP (eval BatchNorm folded at commit, ReLU) with one neighbour per lane and
//              a shuffle max-pool over the neighbours.
//   k_sa2_head set abstraction 2 with its single centre (num_keypoints = 1 => FPS returns point 0), both
//              scales, max-pool, then Linear(256 -> 253) and the [xyz | features] concatenation: one block per
//              cloud, activations in shared memory.
#include "common.cuh"

namespace {

constexpr int FPS_T = 512;       // threads of the sampling kernel (upstream: min(2^floor(log2 N), 512))
constexpr int FPS_MAXPT = 8;     // points per thread -> N <= 4096

__device__ __forceinline__ float pn_dist2(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = ax - bx, dy = ay - by, dz = az - bz;
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__global__ void __launch_bounds__(FPS_T)
k_fps(const float* __restrict__ xyz, int N, int m, float* __restrict__ new_xyz) {
    __shared__ float s_v[FPS_T / 32];
    __shared__ int s_i[FPS_T / 32];
    __shared__ int s_old;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* p = xyz + (size_t)b * N * 3;
    float px[FPS_MAXPT], py[FPS_MAXPT], pz[FPS_MAXPT], temp[FPS_MAXPT];
    bool live[FPS_MAXPT];
#pragma unroll
    for (int i = 0; i < FPS_MAXPT; i++) {
        const int k = tid + i * FPS_T;
        live[i] = false;
        px[i] = py[i] = pz[i] = 0.f;
        temp[i] = 1e10f;
        if (k < N) {
            px[i] = p[k * 3]; py[i] = p[k * 3 + 1]; pz[i] = p[k * 3 + 2];
            const float mag = __fadd_rn(__fadd_rn(__fmul_rn(px[i], px[i]), __fmul_rn(py[i], py[i])), __fmul_rn(pz[i], pz[i]));
            live[i] = mag > 1e-3f;
        }
    }
    int old = 0;
    if (tid == 0) { new_xyz[(size_t)b * m * 3] = p[0]; new_xyz[(size_t)b * m * 3 + 1] = p[1]; new_xyz[(size_t)b * m * 3 + 2] = p[2]; }
    for (int j = 1; j < m; j++) {
        const float ox = p[old * 3], oy = p[old * 3 + 1], oz = p[old * 3 + 2];
        float best = -1.f; int besti = 0;
#pragma unroll
        for (int i = 0; i < FPS_MAXPT; i++) {
            if (live[i]) {
                const float d2 = fminf(pn_dist2(px[i], py[i], pz[i], ox, oy, oz), temp[i]);
                temp[i] = d2;
                if (d2 > best) { best = d2; besti = tid + i * FPS_T; }
            }
        }
        // block arg-max: larger value wins, ties go to the lower thread (threads are compared through their ids)
        int bt = tid;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o), ot = __shfl_xor_sync(0xffffffffu, bt, o);
            if (ov > best || (ov == best && ot < bt)) { best = ov; besti = oi; bt = ot; }
        }
        if (lane == 0) { s_v[warp] = best; s_i[warp] = besti; }
        __syncthreads();
        if (warp == 0) {
            float v = lane < FPS_T / 32 ? s_v[lane] : -2.f;
            int vi = lane < FPS_T / 32 ? s_i[lane] : 0, vt = lane;      // warp order == thread order
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, v, o);
                const int oi = __shfl_xor_sync(0xffffffffu, vi, o), ot = __shfl_xor_sync(0xffffffffu, vt, o);
                if (ov > v || (ov == v && ot < vt)) { v = ov; vi = oi; vt = ot; }
            }
            if (lane == 0) s_old = vi;
        }
        __syncthreads();
        old = s_old;
        if (tid == 0) {
            float* o3 = new_xyz + ((size_t)b * m + j) * 3;
            o3[0] = p[old * 3]; o3[1] = p[old * 3 + 1]; o3[2] = p[old * 3 + 2];
        }
    }
}

// ball query by one warp: indices of the first `ns` points (index order) with d2 < r2, padded with the first hit;
// lane i (< ns) returns the i-th index; 0 everywhere when the ball is empty (upstream's zero-initialised output)
__device__ __forceinline__ int warp_ball_query(const float* __restrict__ pts, int N, float cx, float cy, float cz, float r2, int ns, int lane) {
    int mine = 0, cnt = 0, first = 0;
    for (int base = 0; base < N && cnt < ns; base += 32) {
        const int k = base + lane;
        bool hit = false;
        if (k < N) hit = pn_dist2(cx, cy, cz, pts[k * 3], pts[k * 3 + 1], pts[k * 3 + 2]) < r2;
        unsigned mk = __ballot_sync(0xffffffffu, hit);
        if (mk && cnt == 0) first = base + __ffs(mk) - 1;
        while (mk && cnt < ns) {
            const int src = __ffs(mk) - 1;
            mk &= mk - 1;
            if (lane == cnt) mine = base + src;
            cnt++;
        }
    }
    if (lane >= cnt) mine = first;       // padding (first == 0 when nothing was found)
    return mine;
}

// SA1: xyz (B,N,3) + scalar feature |p| -> feat1 [B][m][96] (scale 0: 32 ch, scale 1: 64 ch), centres new_xyz (B,m,3).
// weights per scale: W1 [C1][4], b1, W2 [C2][C1], b2, W3 [C3][C2], b3 (BatchNorm folded), packed in `wpack`.
template <int C1, int C2, int C3, int NS>
__device__ __forceinline__ void sa1_scale(const float* __restrict__ pts, int N, float cx, float cy, float cz, float radius,
                                          const float* __restrict__ w, float* __restrict__ out, int lane) {
    const int idx = warp_ball_query(pts, N, cx, cy, cz, __fmul_rn(radius, radius), NS, lane);
    const float x = pts[idx * 3], y = pts[idx * 3 + 1], z = pts[idx * 3 + 2];
    const float in[4] = {x - cx, y - cy, z - cz, sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)))};
    const float* W1 = w; const float* B1 = W1 + C1 * 4;
    const float* W2 = B1 + C1; const float* B2 = W2 + C2 * C1;
    const float* W3 = B2 + C2; const float* B3 = W3 + C3 * C2;
    float h1[C1], h2[C2];
#pragma unroll
    for (int o = 0; o < C1; o++) {
        float a = B1[o];
#pragma unroll
        for (int i = 0; i < 4; i++) a = fmaf(W1[o * 4 + i], in[i], a);
        h1[o] = fmaxf(a, 0.f);
    }
#pragma unroll
    for (int o = 0; o < C2; o++) {
        float a = B2[o];
#pragma unroll
        for (int i = 0; i < C1; i++) a = fmaf(W2[o * C1 + i], h1[i], a);
        h2[o] = fmaxf(a, 0.f);
    }
#pragma unroll 4
    for (int o = 0; o < C3; o++) {
        float a = B3[o];
#pragma unroll
        for (int i = 0; i < C2; i++) a = fmaf(W3[o * C2 + i], h2[i], a);
        a = lane < NS ? fmaxf(a, 0.f) : -INFINITY;
#pragma unroll
        for (int s = 16; s; s >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, s));
        if (lane == (o & 31)) out[o] = a;
    }
}

constexpr int SA1_W0 = 16 * 4 + 16 + 16 * 16 + 16 + 32 * 16 + 32;    // 896 floats
constexpr int SA1_W1 = 32 * 4 + 32 + 32 * 32 + 32 + 64 * 32 + 64;    // 3328 floats
__global__ void __launch_bounds__(256)
k_sa1(const float* __restrict__ xyz, int N, const float* __restrict__ new_xyz, int m, const float* __restrict__ wpack,
      float* __restrict__ feat1) {
    __shared__ float s_w[SA1_W0 + SA1_W1];
    for (int i = threadIdx.x; i < SA1_W0 + SA1_W1; i += 256) s_w[i] = wpack[i];
    __syncthreads();
    const int b = blockIdx.y, lane = threadIdx.x & 31, c = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (c >= m) return;
    const float* pts = xyz + (size_t)b * N * 3;
    const float* ctr = new_xyz + ((size_t)b * m + c) * 3;
    const float cx = ctr[0], cy = ctr[1], cz = ctr[2];
    float* out = feat1 + ((size_t)b * m + c) * 96;
    sa1_scale<16, 16, 32, 16>(pts, N, cx, cy, cz, 0.05f, s_w, out, lane);
    sa1_scale<32, 32, 64, 32>(pts, N, cx, cy, cz, 0.1f, s_w + SA1_W0, out + 32, lane);
}

// SA2 (single centre = SA1 centre 0) + Linear head.  Block per cloud, 256 threads.
//   pts1 (B,m,3), feat1 [B][m][96];  scale s: nsample NS_s, layers 99 -> A_s -> B_s -> 128
//   w2pack: per scale W1 [A][99], b1, W2 [Bc][A], b2, W3 [128][Bc], b3;  then Linear W [253][256], b [253]
__global__ void __launch_bounds__(256)
k_sa2_head(const float* __restrict__ pts1, const float* __restrict__ feat1, int m, const float* __restrict__ w2pack,
           float* __restrict__ out) {
    __shared__ int s_idx[48];
    __shared__ float s_xh[48 * 100];     // grouped inputs [48][100] (rel xyz + 96 features), later layer-2 outputs [48][96]
    __shared__ float s_h1[48][64];
    __shared__ float s_pool[256];
    float (*s_x)[100] = reinterpret_cast<float (*)[100]>(s_xh);
    float (*s_h2)[96] = reinterpret_cast<float (*)[96]>(s_xh);
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* pts = pts1 + (size_t)b * m * 3;
    const float cx = pts[0], cy = pts[1], cz = pts[2];
    if (warp == 0) { const int i = warp_ball_query(pts, m, cx, cy, cz, __fmul_rn(0.1f, 0.1f), 16, lane); if (lane < 16) s_idx[lane] = i; }
    if (warp == 1) { const int i = warp_ball_query(pts, m, cx, cy, cz, __fmul_rn(0.2f, 0.2f), 32, lane); s_idx[16 + lane] = i; }
    __syncthreads();
    for (int i = tid; i < 48 * 99; i += 256) {
        const int r = i / 99, c = i % 99, k = s_idx[r];
        s_x[r][c] = c < 3 ? pts[k * 3 + c] - (c == 0 ? cx : c == 1 ? cy : cz) : feat1[((size_t)b * m + k) * 96 + c - 3];
    }
    __syncthreads();
    const int A0 = 64, B0 = 64, A1 = 64, B1 = 96;
    const float* w = w2pack;
    const float* W1a = w; const float* b1a = W1a + A0 * 99; const float* W2a = b1a + A0; const float* b2a = W2a + B0 * A0;
    const float* W3a = b2a + B0; const float* b3a = W3a + 128 * B0;
    const float* W1b = b3a + 128; const float* b1b = W1b + A1 * 99; const float* W2b = b1b + A1; const float* b2b = W2b + B1 * A1;
    const float* W3b = b2b + B1; const float* b3b = W3b + 128 * B1;
    const float* Wl = b3b + 128; const float* bl = Wl + 253 * 256;
    // layer 1 (both scales have 64 outputs): rows 0..15 scale a, 16..47 scale b
    for (int i = tid; i < 48 * 64; i += 256) {
        const int r = i / 64, o = i % 64;
        const float* W = r < 16 ? W1a : W1b;
        float a = (r < 16 ? b1a : b1b)[o];
        for (int c = 0; c < 99; c++) a = fmaf(W[o * 99 + c], s_x[r][c], a);
        s_h1[r][o] = fmaxf(a, 0.f);
    }
    __syncthreads();
    // layer 2: scale a 64 -> 64 (rows 0..15), scale b 64 -> 96 (rows 16..47)
    for (int i = tid; i < 16 * 64 + 32 * 96; i += 256) {
        int r, o; const float* W; float a;
        if (i < 16 * 64) { r = i / 64; o = i % 64; W = W2a + o * 64; a = b2a[o]; }
        else { const int j = i - 16 * 64; r = 16 + j / 96; o = j % 96; W = W2b + o * 64; a = b2b[o]; }
        for (int c = 0; c < 64; c++) a = fmaf(W[c], s_h1[r][c], a);
        s_h2[r][o] = fmaxf(a, 0.f);
    }
    __syncthreads();
    // layer 3 + max-pool over the neighbours: thread = output channel (0..127 scale a, 128..255 scale b)
    {
        const bool sb = tid >= 128;
        const int o = tid & 127, r0 = sb ? 16 : 0, nr = sb ? 32 : 16, K = sb ? 96 : 64;
        const float* W = (sb ? W3b : W3a) + o * K;
        const float bias = (sb ? b3b : b3a)[o];
        float mx = -INFINITY;
        for (int r = r0; r < r0 + nr; r++) {
            float a = bias;
            for (int c = 0; c < K; c++) a = fmaf(W[c], s_h2[r][c], a);
            mx = fmaxf(mx, fmaxf(a, 0.f));
        }
        s_pool[tid] = mx;
    }
    __syncthreads();
    // head: [centre xyz | Linear(256 -> 253)]
    float* ob = out + (size_t)b * 256;
    if (tid < 3) ob[tid] = tid == 0 ? cx : tid == 1 ? cy : cz;
    if (tid < 253) {
        float a = bl[tid];
        for (int c = 0; c < 256; c++) a = fmaf(Wl[tid * 256 + c], s_pool[c], a);
        ob[3 + tid] = a;
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side: fold eval-BatchNorm into the 1x1 convolutions and pack the weights
int idb_pointnet_commit(idb_handle* h) {
    Denoiser& d = h->den;
    d.pn_ready = false;
    if (!d.raw.count("pcEmbedding.Linear.weight")) return IDB_OK;      // optional component
    auto host = [&](const std::string& n, std::vector<float>& v, size_t expect) -> int {
        auto it = d.raw.find(n);
        if (it == d.raw.end()) return idb_fail(h, IDB_ERR_STATE, "missing weight '%s'", n.c_str());
        if (it->second.numel() != expect) return idb_fail(h, IDB_ERR_STATE, "weight '%s' has %zu elements, expected %zu", n.c_str(), it->second.numel(), expect);
        v.resize(expect);
        CUDA_TRY(h, cudaMemcpy(v.data(), it->second.p, expect * sizeof(float), cudaMemcpyDeviceToHost));
        return IDB_OK;
    };
    // conv (index li) + BatchNorm (li + 1) of `prefix` -> folded [Cout][Cin] weights and bias appended to `pack`
    auto fold = [&](const std::string& prefix, int li, int cout, int cin, std::vector<float>& pack) -> int {
        std::vector<float> w, g, bt, mu, var;
        int rc;
        const std::string c = prefix + std::to_string(li) + ".", n = prefix + std::to_string(li + 1) + ".";
        if ((rc = host(c + "weight", w, (size_t)cout * cin))) return rc;
        if ((rc = host(n + "weight", g, cout)) || (rc = host(n + "bias", bt, cout)) || (rc = host(n + "running_mean", mu, cout)) ||
            (rc = host(n + "running_var", var, cout))) return rc;
        for (int o = 0; o < cout; o++) {
            const double s = (double)g[o] / std::sqrt((double)var[o] + 1e-5);
            for (int i = 0; i < cin; i++) pack.push_back((float)(w[(size_t)o * cin + i] * s));
        }
        for (int o = 0; o < cout; o++) {
            const double s = (double)g[o] / std::sqrt((double)var[o] + 1e-5);
            // bias goes right after the layer's weights
            pack.push_back((float)((double)bt[o] - (double)mu[o] * s));
        }
        return IDB_OK;
    };
    std::vector<float> p1, p2;
    int rc;
    const int sa1[2][4] = {{4, 16, 16, 32}, {4, 32, 32, 64}}, sa2[2][4] = {{99, 64, 64, 128}, {99, 64, 96, 128}};
    for (int s = 0; s < 2; s++)
        for (int l = 0; l < 3; l++)
            if ((rc = fold("pcEmbedding.SA_modules.0.mlps." + std::to_string(s) + ".", 3 * l, sa1[s][l + 1], sa1[s][l], p1))) return rc;
    for (int s = 0; s < 2; s++)
        for (int l = 0; l < 3; l++)
            if ((rc = fold("pcEmbedding.SA_modules.1.mlps." + std::to_string(s) + ".", 3 * l, sa2[s][l + 1], sa2[s][l], p2))) return rc;
    std::vector<float> lw, lb;
    if ((rc = host("pcEmbedding.Linear.weight", lw, (size_t)253 * 256)) || (rc = host("pcEmbedding.Linear.bias", lb, 253))) return rc;
    p2.insert(p2.end(), lw.begin(), lw.end());
    p2.insert(p2.end(), lb.begin(), lb.end());
    if ((int)p1.size() != SA1_W0 + SA1_W1) return idb_fail(h, IDB_ERR_STATE, "internal: SA1 pack size %zu", p1.size());
    if ((rc = idb_upload(h, &d.pn_w1, p1.data(), p1.size()))) return rc;
    d.owned.push_back(d.pn_w1);
    if ((rc = idb_upload(h, &d.pn_w2, p2.data(), p2.size()))) return rc;
    d.owned.push_back(d.pn_w2);
    d.pn_ready = true;
    return IDB_OK;
}

extern "C" int idb_pointcloud_embed(idb_handle* h, int B, int P, const float* obj_points, float* pc_embedding, void* stream) {
    IDB_ENTER(h);
    if (!h || !obj_points || !pc_embedding || B <= 0 || P <= 0) return IDB_ERR_ARG;
    Denoiser& d = h->den;
    if (!d.committed || !d.pn_ready) return idb_fail(h, IDB_ERR_STATE, "the point-cloud encoder's weights (pcEmbedding.*) were not loaded / committed");
    const int m = 1024;
    if (P < 512 || P > FPS_T * FPS_MAXPT) return idb_fail(h, IDB_ERR_ARG, "point clouds of 512..%d points are supported (got %d)", FPS_T * FPS_MAXPT, P);
    cudaStream_t st = (cudaStream_t)stream;
    if (B > d.pn_cap) {
        if (d.pn_xyz1) { cudaFree(d.pn_xyz1); cudaFree(d.pn_feat1); d.pn_xyz1 = d.pn_feat1 = nullptr; }
        CUDA_TRY(h, cudaMalloc((void**)&d.pn_xyz1, sizeof(float) * (size_t)B * m * 3));
        CUDA_TRY(h, cudaMalloc((void**)&d.pn_feat1, sizeof(float) * (size_t)B * m * 96));
        d.pn_cap = B;
    }
    k_fps<<<B, FPS_T, 0, st>>>(obj_points, P, m, d.pn_xyz1);
    LAUNCH_CHECK(h);
    k_sa1<<<dim3((m + 7) / 8, B), 256, 0, st>>>(obj_points, P, d.pn_xyz1, m, d.pn_w1, d.pn_feat1);
    LAUNCH_CHECK(h);
    k_sa2_head<<<B, 256, 0, st>>>(d.pn_xyz1, d.pn_feat1, m, d.pn_w2, pc_embedding);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

void idb_pointnet_release(idb_handle* h) {
    Denoiser& d = h->den;
    if (d.pn_xyz1) { cudaFree(d.pn_xyz1); cudaFree(d.pn_feat1); d.pn_xyz1 = d.pn_feat1 = nullptr; }
    d.pn_cap = 0;
    d.pn_ready = false;
}
