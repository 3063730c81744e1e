// Contact-frame correction: ObjProjector.sample (reference model/correction_smpl.py:79-138,
// model/layers.py:271-345, model/sublayers.py:378-419,464-516) and the denoised_fn hook of the
// sampling driver (reference eval_smpl_short.py:84-130).  fp32 throughout.
//
// Frame order inside this file: f = t*B + b (the reference's (T,B,...) flattening).
#include "common.cuh"
#include "body.cuh"
#include "rot.cuh"

struct ProjLayer {
    int cin, cout, ver, P;            // ver 0: shared temporal matrix; ver 2: per-node temporal + spatial
    float *Tm, *A;                    // Tm: [10][10] or [P][10][10];  A: [10][P][P] (ver 2)
    float *W, *b, *Wr, *br;           // BN(eval)-folded 1x1 convs: [cout][cin], [cout]
    float prelu;
};

struct Projector {
    int past = 0, future = 0, n_pre = 0, P = 0, T = 0;
    int variant = 0;                   // 0 = SMPL markers net (n_pre 10, width 32), 1 = skeleton net (n_pre 20, joint stack width 64)
    bool committed = false;
    std::map<std::string, DevTensor> raw;
    std::vector<void*> owned;
    ProjLayer* layers_dev = nullptr;   // 12 layers: relative x4, absolute x4, all x4
    float *dct = nullptr, *idct = nullptr;   // [n_pre][T], [T][n_pre]
    // per-batch workspaces
    int capB = 0;
    float* resid = nullptr;            // [B][9*n_pre*(P+1)]
    // correction context
    int B = 0, cT = 0, cpast = 0, n_obj = 0, n_hand = 0;
    float *hand_pose = nullptr, *betas = nullptr, *obj_points = nullptr;
    int32_t *marker_ids = nullptr, *hand_ids = nullptr;
    float *pose = nullptr, *trans = nullptr, *objRt = nullptr, *verts = nullptr, *normals = nullptr, *objp = nullptr,
          *o2h = nullptr, *markers = nullptr, *pen = nullptr, *dmin = nullptr, *gt_ang = nullptr, *gt_tr = nullptr, *proj_out = nullptr;
    unsigned char *lbl = nullptr, *cond = nullptr;
    int32_t* contact = nullptr;
    std::vector<void*> ctx_owned;
    float *skel_ws = nullptr, *skel_hook_ws = nullptr; int skel_cap = 0, skel_hook_cap = 0;     // skeleton variant workspaces
    // optional decision log (idb_correction_set_log): slot k receives the decisions of the k-th correction step enqueued
    unsigned char* log_cond = nullptr; int32_t* log_contact = nullptr; int log_cap = 0, log_n = 0;
};

namespace {

constexpr int MAXP_SMPL = 68;
constexpr int PROJ_NT = 512;    // threads per projector block: the net is a chain of small latency-bound phases, more warps hide more of it    // 67 markers + the object's own node

// One block per sample: the whole projector runs out of shared memory.  NQ = n_pre (DCT coefficients kept), MAXC = widest
// layer, MAXP = nodes of the joint stack: <10, 32, 68> for the SMPL net (model/correction_smpl.py), <20, 64, 22> for the
// skeleton net (model/correction_skeleton.py: 21 joints + 1, st_gcnns_all 9-64-32-64-9).  select_contact: the SMPL net picks
// the hypothesis of the most-contacted marker (correction_smpl.py:125-136); the skeleton net always reads node 0 (:129).
template <int NQ, int MAXC, int MAXP, int NT>
__global__ void __launch_bounds__(NT)
k_projector(const ProjLayer* __restrict__ layers, const float* __restrict__ dct, const float* __restrict__ idct,
            const float* __restrict__ ang, const float* __restrict__ tr, const float* __restrict__ markers,
            const int32_t* __restrict__ contact, const int32_t* __restrict__ hand_ids, int n_hand,
            float* __restrict__ resid, float* __restrict__ out, int T, int B, int P, int past, int select_contact) {
    extern __shared__ __align__(16) float sm[];
    const int P1 = P + 1;
    float* bufA = sm;                          // [MAXC][NQ][P1]  activations (x / layer output)
    float* bufB = bufA + MAXC * NQ * MAXP;     // [MAXC][NQ][P1]  graph-conv output
    float* s_dct = bufB + MAXC * NQ * MAXP;    // [NQ][T]
    float* s_T = s_dct + NQ * T;               // [NQ][NQ]
    __shared__ int s_sel;
    const int b = blockIdx.x, tid = threadIdx.x;
    float* rs = resid + (size_t)b * 9 * NQ * P1;
    for (int i = tid; i < NQ * T; i += NT) s_dct[i] = dct[i];
    __syncthreads();

    auto run_stack = [&](int l0, int C0, int Pn) {
        // bufA holds x [C0][NQ][Pn]; on exit bufA holds the stack output [9][NQ][Pn]
        for (int li = 0; li < 4; li++) {
            const ProjLayer L = layers[l0 + li];
            const int cin = L.cin, cout = L.cout, npos = NQ * Pn;
            if (L.ver == 0) {
                for (int i = tid; i < NQ * NQ; i += NT) s_T[i] = L.Tm[i];
                __syncthreads();
                for (int it = tid; it < cin * Pn; it += NT) {
                    const int c = it / Pn, p = it % Pn;
                    float xv[NQ];
#pragma unroll
                    for (int t = 0; t < NQ; t++) xv[t] = bufA[(c * NQ + t) * Pn + p];
#pragma unroll
                    for (int q = 0; q < NQ; q++) {
                        float a = 0.f;
#pragma unroll
                        for (int t = 0; t < NQ; t++) a = fmaf(xv[t], s_T[t * NQ + q], a);
                        bufB[(c * NQ + q) * Pn + p] = a;
                    }
                }
                __syncthreads();
            } else {
                for (int it = tid; it < cin * Pn; it += NT) {
                    const int c = it / Pn, p = it % Pn;
                    float xv[NQ];
#pragma unroll
                    for (int t = 0; t < NQ; t++) xv[t] = bufA[(c * NQ + t) * Pn + p];
                    const float* Tv = L.Tm + (size_t)p * NQ * NQ;
#pragma unroll
                    for (int q = 0; q < NQ; q++) {
                        float a = 0.f;
#pragma unroll
                        for (int t = 0; t < NQ; t++) a = fmaf(xv[t], __ldg(Tv + t * NQ + q), a);
                        bufB[(c * NQ + q) * Pn + p] = a;
                    }
                }
                __syncthreads();
                // spatial mix in place, one warp per (c, q) row: g2[w] = sum_v g1[v] A[q][v][w]
                const int warp = tid >> 5, lane = tid & 31;
                for (int row = warp; row < cin * NQ; row += NT / 32) {
                    const int q = row % NQ;
                    float* g = bufB + row * Pn;
                    float r0 = lane < Pn ? g[lane] : 0.f, r1 = lane + 32 < Pn ? g[lane + 32] : 0.f, r2 = lane + 64 < Pn ? g[lane + 64] : 0.f;
                    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
                    const float* Aq = L.A + (size_t)q * Pn * Pn;
                    for (int v = 0; v < Pn; v++) {
                        const float src = v < 32 ? r0 : (v < 64 ? r1 : r2);
                        const float gv = __shfl_sync(0xffffffffu, src, v & 31);
                        const float* Av = Aq + (size_t)v * Pn;
                        if (lane < Pn) o0 = fmaf(gv, __ldg(Av + lane), o0);
                        if (lane + 32 < Pn) o1 = fmaf(gv, __ldg(Av + lane + 32), o1);
                        if (lane + 64 < Pn) o2 = fmaf(gv, __ldg(Av + lane + 64), o2);
                    }
                    __syncwarp();
                    if (lane < Pn) g[lane] = o0;
                    if (lane + 32 < Pn) g[lane + 32] = o1;
                    if (lane + 64 < Pn) g[lane + 64] = o2;
                }
                __syncthreads();
            }
            // position-wise: out = prelu( W g + b  +  Wr x + br )   (BN folded), written over x
            for (int pos = tid; pos < npos; pos += NT) {
                float xv[MAXC], gv[MAXC];
                for (int c = 0; c < cin; c++) { xv[c] = bufA[c * npos + pos]; gv[c] = bufB[c * npos + pos]; }
                for (int co = 0; co < cout; co++) {
                    float a = __ldg(L.b + co), r = __ldg(L.br + co);
                    const float* w = L.W + co * cin;
                    const float* wr = L.Wr + co * cin;
                    for (int c = 0; c < cin; c++) { a = fmaf(__ldg(w + c), gv[c], a); r = fmaf(__ldg(wr + c), xv[c], r); }
                    const float y = a + r;
                    bufA[co * npos + pos] = y >= 0.f ? y : L.prelu * y;
                }
            }
            __syncthreads();
        }
    };

    auto src_frame = [&](int t) { return t < past ? t : past - 1; };  // idx_pad (correction_smpl.py:84)

    // ---- relative stack: object pose relative to each marker, DCT over the padded past
    for (int it = tid; it < 9 * P; it += NT) {
        const int c = it / P, p = it % P;
        float acc[NQ];
#pragma unroll
        for (int q = 0; q < NQ; q++) acc[q] = 0.f;
        for (int t = 0; t < T; t++) {
            const int s = src_frame(t);
            float v;
            if (c < 6) v = ang[((size_t)s * B + b) * 6 + c];
            else v = tr[((size_t)s * B + b) * 3 + (c - 6)] - markers[(((size_t)s * B + b) * P + p) * 3 + (c - 6)];
#pragma unroll
            for (int q = 0; q < NQ; q++) acc[q] = fmaf(s_dct[q * T + t], v, acc[q]);
        }
#pragma unroll
        for (int q = 0; q < NQ; q++) { bufA[(c * NQ + q) * P + p] = acc[q]; rs[(c * NQ + q) * P + p] = acc[q]; }
    }
    __syncthreads();
    run_stack(0, 9, P);
    // obj_multi = [rel + x][:6] | [rel + x][6:9] + DCT(markers)  -> parked in resid at node slots 1..P
    for (int it = tid; it < 9 * P; it += NT) {
        const int c = it / P, p = it % P;
        float ht[NQ];
#pragma unroll
        for (int q = 0; q < NQ; q++) ht[q] = 0.f;
        if (c >= 6)
            for (int t = 0; t < T; t++) {
                const float v = markers[(((size_t)t * B + b) * P + p) * 3 + (c - 6)];
#pragma unroll
                for (int q = 0; q < NQ; q++) ht[q] = fmaf(s_dct[q * T + t], v, ht[q]);
            }
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            const float v = (rs[(c * NQ + q) * P + p] + bufA[(c * NQ + q) * P + p]) + ht[q];
            bufB[(c * NQ + q) * P + p] = v;   // staged; moved below after everyone has read rs
        }
    }
    __syncthreads();
    for (int it = tid; it < 9 * NQ * P; it += NT) {
        const int cq = it / P, p = it % P;
        rs[cq * P1 + 1 + p] = bufB[cq * P + p];
    }
    __syncthreads();
    // ---- absolute stack (single node)
    if (tid < 9) {
        const int c = tid;
        float acc[NQ];
#pragma unroll
        for (int q = 0; q < NQ; q++) acc[q] = 0.f;
        for (int t = 0; t < T; t++) {
            const int s = src_frame(t);
            const float v = c < 6 ? ang[((size_t)s * B + b) * 6 + c] : tr[((size_t)s * B + b) * 3 + (c - 6)];
#pragma unroll
            for (int q = 0; q < NQ; q++) acc[q] = fmaf(s_dct[q * T + t], v, acc[q]);
        }
#pragma unroll
        for (int q = 0; q < NQ; q++) { bufA[c * NQ + q] = acc[q]; rs[(c * NQ + q) * P1] = acc[q]; }
    }
    __syncthreads();
    run_stack(4, 9, 1);
    if (tid < 9 * NQ) rs[tid * P1] += bufA[tid];
    __syncthreads();
    // ---- joint stack over P+1 nodes
    for (int it = tid; it < 9 * NQ * P1; it += NT) bufA[it] = rs[it];
    __syncthreads();
    run_stack(8, 9, P1);
    // ---- hypothesis selection (correction_smpl.py:125-136) + inverse DCT of that column only
    if (tid == 0) {
        long long csum = 0;
        if (select_contact) for (int p = 0; p < P; p++) csum += contact[(size_t)b * P + p];
        int sel = 0;
        if (csum > 0) {
            float best = -INFINITY;
            int bi = 0;
            for (int p = 0; p < P; p++) {
                float v = (float)contact[(size_t)b * P + p];
                for (int k = 0; k < n_hand; k++) if (hand_ids[k] == p) { v += 0.5f; break; }
                if (v > best) { best = v; bi = p; }   // argmax: first maximum
            }
            sel = 1 + bi;
        }
        s_sel = sel;
    }
    __syncthreads();
    const int sel = s_sel;
    for (int it = tid; it < T * 9; it += NT) {
        const int t = it / 9, c = it % 9;
        float a = 0.f;
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            const float v = rs[(c * NQ + q) * P1 + sel] + bufA[(c * NQ + q) * P1 + sel];
            a = fmaf(idct[t * NQ + q], v, a);
        }
        out[((size_t)t * B + b) * 9 + c] = a;
    }
}

// ---- denoised_fn pieces --------------------------------------------------------------------

// x0 (B,1,C,T) -> per frame f = t*B + b: pose156 = [aa(22 joints) | hand90], trans, object R|t
__global__ void k_corr_prepare(const float* __restrict__ x0, const float* __restrict__ hand, float* __restrict__ pose,
                               float* __restrict__ trans, float* __restrict__ objRt, int B, int T, int C) {
    const int f = blockIdx.x, t = f / B, b = f % B, tid = threadIdx.x;
    const float* xb = x0 + (size_t)b * C * T + t;   // channel c at xb[c*T]
    if (tid < 22) {
        float d6[6], R[9], aa[3];
        for (int k = 0; k < 6; k++) d6[k] = xb[(size_t)(tid * 6 + k) * T];
        idb_rot6d_to_matrix(d6, R);
        idb_matrix_to_axis_angle(R, aa);
        pose[(size_t)f * 156 + tid * 3] = aa[0]; pose[(size_t)f * 156 + tid * 3 + 1] = aa[1]; pose[(size_t)f * 156 + tid * 3 + 2] = aa[2];
    } else if (tid == 22) {
        float d6[6], R[9];
        for (int k = 0; k < 6; k++) d6[k] = xb[(size_t)(135 + k) * T];
        idb_rot6d_to_matrix(d6, R);
        for (int k = 0; k < 9; k++) objRt[(size_t)f * 12 + k] = R[k];
        for (int k = 0; k < 3; k++) objRt[(size_t)f * 12 + 9 + k] = xb[(size_t)(141 + k) * T];
    } else if (tid == 23) {
        for (int k = 0; k < 3; k++) trans[(size_t)f * 3 + k] = xb[(size_t)(132 + k) * T];
    }
    for (int k = tid; k < 90; k += blockDim.x) pose[(size_t)f * 156 + 66 + k] = hand[(size_t)f * 90 + k];
}

// obj_points_pred = P R^T + t   (eval_smpl_short.py:107)
__global__ void k_obj_points(const float* __restrict__ pts, const float* __restrict__ objRt, float* __restrict__ out, int B, int Pn) {
    const int f = blockIdx.y, b = f % B, p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= Pn) return;
    const float* R = objRt + (size_t)f * 12;
    const float x = pts[((size_t)b * Pn + p) * 3], y = pts[((size_t)b * Pn + p) * 3 + 1], z = pts[((size_t)b * Pn + p) * 3 + 2];
    float* o = out + ((size_t)f * Pn + p) * 3;
    o[0] = (x * R[0] + y * R[1] + z * R[2]) + R[9];
    o[1] = (x * R[3] + y * R[4] + z * R[5]) + R[10];
    o[2] = (x * R[6] + y * R[7] + z * R[8]) + R[11];
}

// Per frame: markers gather, penetration loss mean, marker<->object min distance, contact labels.
__global__ void __launch_bounds__(256)
k_frame_stats(const float* __restrict__ verts, const int32_t* __restrict__ marker_ids, const float* __restrict__ objp,
              const float* __restrict__ o2h, float* __restrict__ markers, float* __restrict__ pen, float* __restrict__ dmin,
              unsigned char* __restrict__ lbl, int V, int Pn, int P) {
    __shared__ float s_m[MAXP_SMPL * 3];
    __shared__ float s_red[256];
    __shared__ unsigned int s_lbl[MAXP_SMPL];
    __shared__ float s_min[8];
    const int f = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < P * 3; i += 256) {
        const float v = verts[((size_t)f * V + marker_ids[i / 3]) * 3 + i % 3];
        s_m[i] = v;
        markers[(size_t)f * P * 3 + i] = v;
    }
    if (tid < P) s_lbl[tid] = 0;
    __syncthreads();
    float psum = 0.f, mn = INFINITY;
    for (int p = tid; p < Pn; p += 256) {
        const float d = o2h[(size_t)f * Pn + p];
        psum += d < 0.f ? fabsf(d) * 20.0f : 0.0f;   // w = 20 where penetrating, 0 elsewhere (:113-118)
        const float x = objp[((size_t)f * Pn + p) * 3], y = objp[((size_t)f * Pn + p) * 3 + 1], z = objp[((size_t)f * Pn + p) * 3 + 2];
        for (int m = 0; m < P; m++) {
            const float dx = s_m[m * 3] - x, dy = s_m[m * 3 + 1] - y, dz = s_m[m * 3 + 2] - z;
            const float dd = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            mn = fminf(mn, dd);
            if (dd < 0.02f) s_lbl[m] = 1u;   // benign race: every writer stores 1
        }
    }
    s_red[tid] = psum;
    mn = -warp_max(-mn);
    if ((tid & 31) == 0) s_min[tid >> 5] = mn;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (tid < s) s_red[tid] += s_red[tid + s]; __syncthreads(); }
    if (tid == 0) {
        pen[f] = s_red[0] / (float)Pn;
        float m = s_min[0];
        for (int i = 1; i < 8; i++) m = fminf(m, s_min[i]);
        dmin[f] = m;
    }
    if (tid < P) lbl[(size_t)f * P + tid] = (unsigned char)s_lbl[tid];
}

__global__ void k_decide(const float* __restrict__ pen, const float* __restrict__ dmin, const unsigned char* __restrict__ lbl,
                         unsigned char* __restrict__ cond, int32_t* __restrict__ contact, int T, int B, int P, int past) {
    const int b = blockIdx.x, tid = threadIdx.x;
    if (tid < P) {
        int c = 0;
        for (int t = past; t < T; t++) c += lbl[((size_t)t * B + b) * P + tid];
        contact[(size_t)b * P + tid] = c;
    }
    if (tid == 0) {
        float ps = 0.f, ds = 0.f;
        for (int t = past; t < T; t++) ps += pen[t * B + b];
        for (int t = 0; t < T; t++) ds += dmin[t * B + b];
        const bool ok = (ps / (float)(T - past) < 0.002f) && (ds / (float)T < 0.02f);
        cond[b] = ok ? 0 : 1;
    }
}

// gt (B,1,C,T) -> obj 6D (T,B,6) and trans (T,B,3)
__global__ void k_gt_obj(const float* __restrict__ gt, float* __restrict__ ang, float* __restrict__ tr, int B, int T, int C) {
    const int f = blockIdx.x, t = f / B, b = f % B, k = threadIdx.x;
    if (k < 6) ang[(size_t)f * 6 + k] = gt[((size_t)b * C + 135 + k) * T + t];
    else if (k < 9) tr[(size_t)f * 3 + (k - 6)] = gt[((size_t)b * C + 141 + (k - 6)) * T + t];
}

// x_ = cat[body, obj_proj];  x_ = a x + (1-a) x_;  x[condition] = x_[condition]   (:127-129)
__global__ void k_blend(float* x, const float* __restrict__ proj, const unsigned char* __restrict__ cond, float a, int B, int T, int C) {
    const size_t n = (size_t)B * C * T;
    const float a1 = 1.0f - a;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const int t = e % T, c = (e / T) % C, b = e / ((size_t)T * C);
        if (!cond[b]) continue;
        const float xv = x[e];
        const float other = c < 135 ? xv : proj[((size_t)t * B + b) * 9 + (c - 135)];
        x[e] = __fadd_rn(__fmul_rn(a, xv), __fmul_rn(a1, other));
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
void idb_projector_release(idb_handle* h) {
    if (!h->proj) return;
    h->epoch++;
    Projector& p = *h->proj;
    for (auto& kv : p.raw) cudaFree(kv.second.p);
    for (void* q : p.owned) cudaFree(q);
    for (void* q : p.ctx_owned) cudaFree(q);
    if (p.resid) cudaFree(p.resid);
    if (p.hand_ids) cudaFree(p.hand_ids);
    if (p.skel_ws) cudaFree(p.skel_ws);
    if (p.skel_hook_ws) cudaFree(p.skel_hook_ws);
    delete h->proj;
    h->proj = nullptr;
}

extern "C" int idb_projector_init(idb_handle* h, int past_len, int future_len, int n_pre, int n_markers) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    if (n_pre != 10) return idb_fail(h, IDB_ERR_ARG, "n_pre (dct) must be 10 for the SMPL correction net (20: idb_projector_init_skeleton)");
    if (n_markers + 1 > MAXP_SMPL || n_markers < 1) return idb_fail(h, IDB_ERR_ARG, "n_markers must be in 1..67");
    if (past_len < 1 || future_len < 0) return IDB_ERR_ARG;
    idb_projector_release(h);
    h->proj = new Projector();
    Projector& p = *h->proj;
    p.past = past_len; p.future = future_len; p.n_pre = n_pre; p.P = n_markers; p.T = past_len + future_len;
    return IDB_OK;
}

/* skeleton correction net (model/correction_skeleton.py:8-53): n_pre = 20, joint stack 9-64-32-64-9 over n_joints + 1 nodes */
extern "C" int idb_projector_init_skeleton(idb_handle* h, int past_len, int future_len, int n_joints) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    if (n_joints < 1 || n_joints + 1 > 22) return idb_fail(h, IDB_ERR_ARG, "n_joints must be in 1..21");
    if (past_len < 1 || future_len < 0) return IDB_ERR_ARG;
    idb_projector_release(h);
    h->proj = new Projector();
    Projector& p = *h->proj;
    p.variant = 1;
    p.past = past_len; p.future = future_len; p.n_pre = 20; p.P = n_joints; p.T = past_len + future_len;
    return IDB_OK;
}

extern "C" int idb_projector_load(idb_handle* h, const char* name, const float* data, const int64_t* shape, int ndim) {
    IDB_ENTER(h);
    if (!h || !name || !data) return IDB_ERR_ARG;
    if (!h->proj) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init first");
    std::string s(name);
    if (s.rfind("st_gcnns", 0) != 0 || s.find("num_batches_tracked") != std::string::npos) return IDB_OK;
    Projector& p = *h->proj;
    DevTensor t;
    t.shape.assign(shape, shape + ndim);
    auto it = p.raw.find(s);
    if (it != p.raw.end()) { cudaFree(it->second.p); p.raw.erase(it); }
    int rc = idb_upload(h, &t.p, data, t.numel());
    if (rc) return rc;
    p.raw[s] = t;
    p.committed = false;
    return IDB_OK;
}

extern "C" int idb_projector_commit(idb_handle* h) {
    IDB_ENTER(h);
    if (!h || !h->proj) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init first");
    Projector& p = *h->proj;
    for (void* q : p.owned) cudaFree(q);
    p.owned.clear();
    auto hostof = [&](const std::string& n, std::vector<float>& out) -> int {
        auto it = p.raw.find(n);
        if (it == p.raw.end()) return idb_fail(h, IDB_ERR_STATE, "missing projector weight '%s'", n.c_str());
        out.resize(it->second.numel());
        cudaMemcpy(out.data(), it->second.p, out.size() * 4, cudaMemcpyDeviceToHost);
        return 0;
    };
    auto up = [&](const std::vector<float>& v, float** dst) -> int {
        CUDA_TRY(h, cudaMalloc((void**)dst, v.size() * 4 + 4));
        CUDA_TRY(h, cudaMemcpy(*dst, v.data(), v.size() * 4, cudaMemcpyHostToDevice));
        p.owned.push_back(*dst);
        return 0;
    };
    const char* stacks[3] = {"st_gcnns_relative.", "st_gcnns.", "st_gcnns_all."};
    const int nodes[3] = {p.P, 1, p.P + 1};
    const int NQ = p.n_pre;
    // layer widths (model/correction_smpl.py:18-50; model/correction_skeleton.py:13-50: the joint stack is 9-64-32-64-9)
    const int chans_std[5] = {9, 32, 16, 32, 9}, chans_wide[5] = {9, 64, 32, 64, 9};
    std::vector<ProjLayer> L(12);
    int rc;
    for (int s = 0; s < 3; s++)
        for (int i = 0; i < 4; i++) {
            ProjLayer& l = L[s * 4 + i];
            const std::string pre = std::string(stacks[s]) + std::to_string(i) + ".";
            const int* chans = (p.variant == 1 && s == 2) ? chans_wide : chans_std;
            l.cin = chans[i]; l.cout = chans[i + 1]; l.ver = s == 2 ? 2 : 0; l.P = nodes[s]; l.A = nullptr;
            std::vector<float> Tm, A, W, b, g, be, mu, var, Wr, br, gr, ber, mur, varr, pr;
            if ((rc = hostof(pre + "gcn.T", Tm))) return rc;
            const size_t wantT = l.ver == 2 ? (size_t)l.P * NQ * NQ : (size_t)NQ * NQ;
            if (Tm.size() != wantT) return idb_fail(h, IDB_ERR_STATE, "'%sgcn.T' has the wrong shape", pre.c_str());
            if ((rc = up(Tm, &l.Tm))) return rc;
            if (l.ver == 2) {
                if ((rc = hostof(pre + "gcn.A", A))) return rc;
                if (A.size() != (size_t)NQ * l.P * l.P) return idb_fail(h, IDB_ERR_STATE, "'%sgcn.A' has the wrong shape", pre.c_str());
                if ((rc = up(A, &l.A))) return rc;
            }
            if ((rc = hostof(pre + "tcn.0.weight", W)) || (rc = hostof(pre + "tcn.0.bias", b)) || (rc = hostof(pre + "tcn.1.weight", g)) ||
                (rc = hostof(pre + "tcn.1.bias", be)) || (rc = hostof(pre + "tcn.1.running_mean", mu)) || (rc = hostof(pre + "tcn.1.running_var", var)) ||
                (rc = hostof(pre + "residual.0.weight", Wr)) || (rc = hostof(pre + "residual.0.bias", br)) || (rc = hostof(pre + "residual.1.weight", gr)) ||
                (rc = hostof(pre + "residual.1.bias", ber)) || (rc = hostof(pre + "residual.1.running_mean", mur)) ||
                (rc = hostof(pre + "residual.1.running_var", varr)) || (rc = hostof(pre + "prelu.weight", pr)))
                return rc;
            if (W.size() != (size_t)l.cin * l.cout || Wr.size() != W.size()) return idb_fail(h, IDB_ERR_STATE, "'%s' conv has the wrong shape", pre.c_str());
            // fold eval-mode BatchNorm (eps 1e-5) into the 1x1 convs
            for (int co = 0; co < l.cout; co++) {
                const float s1 = g[co] / std::sqrt(var[co] + 1e-5f), s2 = gr[co] / std::sqrt(varr[co] + 1e-5f);
                for (int c = 0; c < l.cin; c++) { W[co * l.cin + c] *= s1; Wr[co * l.cin + c] *= s2; }
                b[co] = (b[co] - mu[co]) * s1 + be[co];
                br[co] = (br[co] - mur[co]) * s2 + ber[co];
            }
            if ((rc = up(W, &l.W)) || (rc = up(b, &l.b)) || (rc = up(Wr, &l.Wr)) || (rc = up(br, &l.br))) return rc;
            l.prelu = pr[0];
        }
    CUDA_TRY(h, cudaMalloc((void**)&p.layers_dev, sizeof(ProjLayer) * 12));
    p.owned.push_back(p.layers_dev);
    CUDA_TRY(h, cudaMemcpy(p.layers_dev, L.data(), sizeof(ProjLayer) * 12, cudaMemcpyHostToDevice));
    // DCT-II matrix (correction_smpl.py:55-67) in float64, cast to float; inverse = transpose
    const int T = p.T;
    std::vector<float> dct((size_t)NQ * T), idct((size_t)T * NQ);
    for (int k = 0; k < NQ; k++)
        for (int i = 0; i < T; i++) {
            const double w = k == 0 ? std::sqrt(1.0 / T) : std::sqrt(2.0 / T);
            const double v = w * std::cos(M_PI * (i + 0.5) * k / T);
            dct[(size_t)k * T + i] = (float)v;
            idct[(size_t)i * NQ + k] = (float)v;
        }
    if ((rc = up(dct, &p.dct)) || (rc = up(idct, &p.idct))) return rc;
    // per-function, per-device opt-in: always the device maximum (a smaller value set by another handle must not undercut it)
    // (the kernels also hold a few bytes of static shared memory: the dynamic limit is the device maximum minus that)
    cudaFuncAttributes fa;
    CUDA_TRY(h, cudaFuncGetAttributes(&fa, k_projector<10, 32, 68, PROJ_NT>));
    CUDA_TRY(h, cudaFuncSetAttribute(k_projector<10, 32, 68, PROJ_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - (int)fa.sharedSizeBytes));
    CUDA_TRY(h, cudaFuncGetAttributes(&fa, k_projector<20, 64, 22, PROJ_NT>));
    CUDA_TRY(h, cudaFuncSetAttribute(k_projector<20, 64, 22, PROJ_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - (int)fa.sharedSizeBytes));
    p.committed = true;
    h->epoch++;
    return IDB_OK;
}

static int projector_run(idb_handle* h, int T, int B, const float* ang, const float* tr, const float* markers,
                         const int32_t* contact, float* out, cudaStream_t st) {
    Projector& p = *h->proj;
    if (!p.committed) return idb_fail(h, IDB_ERR_STATE, "idb_projector_commit first");
    if (T != p.T) return idb_fail(h, IDB_ERR_ARG, "T must equal past_len + future_len of the projector (%d)", p.T);
    const int NQ = p.n_pre;
    if (B > p.capB) {
        h->epoch++;
        if (p.resid) cudaFree(p.resid);
        CUDA_TRY(h, cudaMalloc((void**)&p.resid, sizeof(float) * (size_t)B * 9 * NQ * (p.P + 1)));
        p.capB = B;
    }
    if (p.variant == 0) {
        const size_t smem = sizeof(float) * ((size_t)2 * 32 * 10 * 68 + NQ * T + NQ * NQ);
        k_projector<10, 32, 68, PROJ_NT><<<B, PROJ_NT, smem, st>>>(p.layers_dev, p.dct, p.idct, ang, tr, markers, contact, p.hand_ids, p.n_hand, p.resid, out,
                                                      T, B, p.P, p.past, 1);
    } else {
        const size_t smem = sizeof(float) * ((size_t)2 * 64 * 20 * 22 + NQ * T + NQ * NQ);
        k_projector<20, 64, 22, PROJ_NT><<<B, PROJ_NT, smem, st>>>(p.layers_dev, p.dct, p.idct, ang, tr, markers, nullptr, nullptr, 0, p.resid, out,
                                                      T, B, p.P, p.past, 0);
    }
    LAUNCH_CHECK(h);
    return IDB_OK;
}

extern "C" int idb_projector_set_hand_markers(idb_handle* h, const int32_t* ids, int n) {
    IDB_ENTER(h);
    if (!h || !ids || n < 0 || n > 64) return IDB_ERR_ARG;
    if (!h->proj) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init first");
    Projector& p = *h->proj;
    if (!p.hand_ids) CUDA_TRY(h, cudaMalloc((void**)&p.hand_ids, 64 * sizeof(int32_t)));
    CUDA_TRY(h, cudaMemcpy(p.hand_ids, ids, (size_t)n * 4, cudaMemcpyDefault));
    if (p.n_hand != n) h->epoch++;
    p.n_hand = n;
    return IDB_OK;
}

extern "C" int idb_projector_sample(idb_handle* h, int T, int B, const float* obj_angles, const float* obj_trans,
                                    const float* markers, const int32_t* contact, float* out, void* stream) {
    IDB_ENTER(h);
    if (!h || !obj_angles || !obj_trans || !markers || !contact || !out) return IDB_ERR_ARG;
    if (!h->proj) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init first");
    if (!h->proj->hand_ids) return idb_fail(h, IDB_ERR_STATE, "idb_projector_set_hand_markers first");
    return projector_run(h, T, B, obj_angles, obj_trans, markers, contact, out, (cudaStream_t)stream);
}

extern "C" int idb_correction_bind(idb_handle* h, int B, int T, int past_len, int n_obj_points, const float* hand_pose,
                                   const float* betas, const float* obj_points, const int32_t* marker_ids,
                                   const int32_t* hand_marker_ids, int n_hand, void* stream) {
    IDB_ENTER(h);
    if (!h || !hand_pose || !betas || !obj_points || !marker_ids || !hand_marker_ids) return IDB_ERR_ARG;
    if (!h->proj) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init first");
    if (!h->body) return idb_fail(h, IDB_ERR_STATE, "idb_body_init first");
    Projector& p = *h->proj;
    BodyModel& m = *h->body;
    if (m.J != 52 || m.NB != 10) return idb_fail(h, IDB_ERR_ARG, "the correction hook expects SMPL-H (52 joints, 10 betas)");
    cudaStream_t st = (cudaStream_t)stream;
    const int F = T * B, P = p.P, V = m.V;
    if (B != p.B || T != p.cT || n_obj_points != p.n_obj) {
        h->epoch++;
        for (void* q : p.ctx_owned) cudaFree(q);
        p.ctx_owned.clear();
        auto A = [&](void** ptr, size_t bytes) {
            cudaError_t e = cudaMalloc(ptr, bytes ? bytes : 4);
            if (e == cudaSuccess) p.ctx_owned.push_back(*ptr);
            return e;
        };
        CUDA_TRY(h, A((void**)&p.hand_pose, (size_t)F * 90 * 4)); CUDA_TRY(h, A((void**)&p.betas, (size_t)F * 10 * 4));
        CUDA_TRY(h, A((void**)&p.obj_points, (size_t)B * n_obj_points * 3 * 4)); CUDA_TRY(h, A((void**)&p.marker_ids, (size_t)P * 4));
        CUDA_TRY(h, A((void**)&p.pose, (size_t)F * 156 * 4)); CUDA_TRY(h, A((void**)&p.trans, (size_t)F * 3 * 4));
        CUDA_TRY(h, A((void**)&p.objRt, (size_t)F * 12 * 4)); CUDA_TRY(h, A((void**)&p.verts, (size_t)F * V * 3 * 4));
        CUDA_TRY(h, A((void**)&p.normals, (size_t)F * V * 3 * 4)); CUDA_TRY(h, A((void**)&p.objp, (size_t)F * n_obj_points * 3 * 4));
        CUDA_TRY(h, A((void**)&p.o2h, (size_t)F * n_obj_points * 4)); CUDA_TRY(h, A((void**)&p.markers, (size_t)F * P * 3 * 4));
        CUDA_TRY(h, A((void**)&p.pen, (size_t)F * 4)); CUDA_TRY(h, A((void**)&p.dmin, (size_t)F * 4));
        CUDA_TRY(h, A((void**)&p.lbl, (size_t)F * P)); CUDA_TRY(h, A((void**)&p.cond, (size_t)B));
        CUDA_TRY(h, A((void**)&p.contact, (size_t)B * P * 4)); CUDA_TRY(h, A((void**)&p.gt_ang, (size_t)F * 6 * 4));
        CUDA_TRY(h, A((void**)&p.gt_tr, (size_t)F * 3 * 4)); CUDA_TRY(h, A((void**)&p.proj_out, (size_t)F * 9 * 4));
        p.B = B; p.cT = T; p.n_obj = n_obj_points;
    }
    if (p.cpast != past_len) h->epoch++;   // kernel parameter of the captured correction steps
    p.cpast = past_len;
    { int rc = idb_projector_set_hand_markers(h, hand_marker_ids, n_hand); if (rc) return rc; }
    CUDA_TRY(h, cudaMemcpyAsync(p.hand_pose, hand_pose, (size_t)F * 90 * 4, cudaMemcpyDefault, st));
    CUDA_TRY(h, cudaMemcpyAsync(p.betas, betas, (size_t)F * 10 * 4, cudaMemcpyDefault, st));
    CUDA_TRY(h, cudaMemcpyAsync(p.obj_points, obj_points, (size_t)B * n_obj_points * 3 * 4, cudaMemcpyDefault, st));
    CUDA_TRY(h, cudaMemcpyAsync(p.marker_ids, marker_ids, (size_t)P * 4, cudaMemcpyDefault, st));
    return IDB_OK;
}

// Grows every workspace a correction step needs BEFORE a stream capture starts (no allocation may happen inside one).
extern "C" int idb_skeleton_correction_apply(idb_handle* h, int B, int T, int n_points, float* x0, const float* gt, const float* zero_pose_obj,
                                             int t, void* stream);
int idb_correction_prepare(idb_handle* h, int B, int T) {
    if (h->proj && h->proj->variant == 1) {
        // skeleton hook: run it once outside any capture on a scratch sample so that every workspace has its final size
        Projector& p = *h->proj;
        const idb_denoiser_config& c = h->den.cfg;
        if (c.variant != 1 || !h->den.zero_pose) return idb_fail(h, IDB_ERR_STATE, "the skeleton correction hook needs the skeleton denoiser bound");
        const int F = T * B;
        if (F <= p.skel_hook_cap && F <= p.skel_cap && B <= p.capB) return IDB_OK;
        const size_t n = (size_t)B * (c.c_body + c.c_obj + c.c_extra) * T;
        float* tmp = nullptr;
        CUDA_TRY(h, cudaMalloc((void**)&tmp, n * sizeof(float)));
        cudaMemset(tmp, 0, n * sizeof(float));
        int rc = idb_skeleton_correction_apply(h, B, T, c.n_points, tmp, tmp, h->den.zero_pose, 0, nullptr);
        cudaDeviceSynchronize();
        cudaFree(tmp);
        return rc;
    }
    if (!h->proj || !h->proj->B) return idb_fail(h, IDB_ERR_STATE, "idb_correction_bind first");
    if (!h->body) return idb_fail(h, IDB_ERR_STATE, "idb_body_init first");
    Projector& p = *h->proj;
    if (p.B != B || p.cT != T) return idb_fail(h, IDB_ERR_STATE, "correction bound for B=%d, T=%d but the denoiser for B=%d, T=%d", p.B, p.cT, B, T);
    int rc = idb_body_workspace(h, p.cT * p.B);
    if (rc) return rc;
    if (p.B > p.capB) {
        h->epoch++;
        if (p.resid) cudaFree(p.resid);
        CUDA_TRY(h, cudaMalloc((void**)&p.resid, sizeof(float) * (size_t)p.B * 9 * p.n_pre * (p.P + 1)));
        p.capB = p.B;
    }
    return IDB_OK;
}

int idb_correction_apply_dev(idb_handle* h, float* x0, const float* gt, int t, cudaStream_t st) {
    if (h->proj && h->proj->variant == 1) {   // skeleton model: eval_skeleton.py's hook on the bound batch
        if (!gt) return idb_fail(h, IDB_ERR_ARG, "the correction hook needs the inpainted motion (gt)");
        return idb_skeleton_correction_apply(h, h->den.B, h->den.T, h->den.cfg.n_points, x0, gt, h->den.zero_pose, t, (void*)st);
    }
    if (!h->proj || !h->proj->B) return idb_fail(h, IDB_ERR_STATE, "idb_correction_bind first");
    if (!gt) return idb_fail(h, IDB_ERR_ARG, "the correction hook needs the inpainted motion (gt)");
    Projector& p = *h->proj;
    BodyModel& m = *h->body;
    const int B = p.B, T = p.cT, F = T * B, C = 144, P = p.P, Pn = p.n_obj;
    int rc;
    k_corr_prepare<<<F, 32, 0, st>>>(x0, p.hand_pose, p.pose, p.trans, p.objRt, B, T, C);
    LAUNCH_CHECK(h);
    if ((rc = idb_smplh_lbs(h, F, p.pose, p.betas, p.trans, p.verts, nullptr, st))) return rc;
    if ((rc = idb_vertex_normals(h, F, p.verts, p.normals, st))) return rc;
    k_obj_points<<<dim3((Pn + 255) / 256, F), 256, 0, st>>>(p.obj_points, p.objRt, p.objp, B, Pn);
    LAUNCH_CHECK(h);
    if ((rc = idb_signed_nn(h, F, Pn, m.V, p.objp, p.verts, p.normals, p.o2h, nullptr, nullptr, st))) return rc;
    k_frame_stats<<<F, 256, 0, st>>>(p.verts, p.marker_ids, p.objp, p.o2h, p.markers, p.pen, p.dmin, p.lbl, m.V, Pn, P);
    LAUNCH_CHECK(h);
    k_decide<<<B, 128, 0, st>>>(p.pen, p.dmin, p.lbl, p.cond, p.contact, T, B, P, p.cpast);
    LAUNCH_CHECK(h);
    if (p.log_cond && p.log_n < p.log_cap) {     // decision log for the parity tests of the in-loop path
        CUDA_TRY(h, cudaMemcpyAsync(p.log_cond + (size_t)p.log_n * B, p.cond, (size_t)B, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(h, cudaMemcpyAsync(p.log_contact + (size_t)p.log_n * B * P, p.contact, (size_t)B * P * 4, cudaMemcpyDeviceToDevice, st));
        p.log_n++;
    }
    k_gt_obj<<<F, 32, 0, st>>>(gt, p.gt_ang, p.gt_tr, B, T, C);
    LAUNCH_CHECK(h);
    if ((rc = projector_run(h, T, B, p.gt_ang, p.gt_tr, p.markers, p.contact, p.proj_out, st))) return rc;
    // t[0] / 1000 in float32 (torch true-divides the int64 tensor by 1000 -> float32)
    const float a = (float)t / 1000.0f;
    k_blend<<<132 * 2, 256, 0, st>>>(x0, p.proj_out, p.cond, a, B, T, C);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

// ---- skeleton variant (model/correction_skeleton.py:84-135, eval_skeleton.py:80-111) ------------------------------------
namespace {
// quaternion xyzw (T,B,4) -> rotation 6D (first two rows of quaternion_to_matrix on (w,x,y,z)), correction_skeleton.py:89-90
__global__ void k_quat_to_6d(const float* __restrict__ quat, float* __restrict__ ang6, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float q[4] = {quat[(size_t)i * 4 + 3], quat[(size_t)i * 4], quat[(size_t)i * 4 + 1], quat[(size_t)i * 4 + 2]};
    float R[9];
    idb_quaternion_to_matrix(q, R);
    for (int e = 0; e < 6; e++) ang6[(size_t)i * 6 + e] = R[e];
}
// projector output (T,B,9) = [6D | trans] -> quaternion xyzw (T,B,4), trans (T,B,3)   (:132-135)
__global__ void k_proj_to_quat(const float* __restrict__ res, float* __restrict__ quat, float* __restrict__ trans, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float R[9], q[4];
    idb_rot6d_to_matrix(res + (size_t)i * 9, R);
    idb_matrix_to_quaternion(R, q);
    quat[(size_t)i * 4] = q[1]; quat[(size_t)i * 4 + 1] = q[2]; quat[(size_t)i * 4 + 2] = q[3]; quat[(size_t)i * 4 + 3] = q[0];
    for (int e = 0; e < 3; e++) trans[(size_t)i * 3 + e] = res[(size_t)i * 9 + 6 + e];
}
// x (B,1,C,T), C = 3 Jn + 3 Np + 7: gathers of the hook's inputs.  which 0: joints (T,B,Jn,3) from x; 1: pose [trans3 | quat4] of gt
__global__ void k_skel_gather(const float* __restrict__ x, float* __restrict__ joints, const float* __restrict__ gt, float* __restrict__ gt_trans,
                              float* __restrict__ gt_quat, int B, int T, int C, int Jn) {
    const int f = blockIdx.x, t = f / B, b = f % B;
    for (int i = threadIdx.x; i < Jn * 3; i += blockDim.x) joints[(size_t)f * Jn * 3 + i] = x[((size_t)b * C + i) * T + t];
    if (threadIdx.x < 7) {
        const float v = gt[((size_t)b * C + (C - 7) + threadIdx.x) * T + t];
        if (threadIdx.x < 3) gt_trans[(size_t)f * 3 + threadIdx.x] = v; else gt_quat[(size_t)f * 4 + threadIdx.x - 3] = v;
    }
}
// x = a x + (1 - a) [body | calc_obj_pred(pose_proj, zero_pose_obj) | pose_proj]   for EVERY sample (eval_skeleton.py:106-111)
__global__ void k_skel_blend(float* __restrict__ x, const float* __restrict__ quat, const float* __restrict__ trans,
                             const float* __restrict__ zero_pose, float a, int B, int T, int C, int Jn, int Np) {
    const int f = blockIdx.x, t = f / B, b = f % B;
    const float a1 = 1.0f - a;
    __shared__ float R[9];
    __shared__ float pose[7];
    if (threadIdx.x == 0) {
        const float* qq = quat + (size_t)f * 4;
        const float q[4] = {qq[3], qq[0], qq[1], qq[2]};          // calc_obj_pred: xyzw -> wxyz, un-normalised
        float Rl[9];
        idb_quaternion_to_matrix(q, Rl);
        for (int e = 0; e < 9; e++) R[e] = Rl[e];
        for (int e = 0; e < 3; e++) pose[e] = trans[(size_t)f * 3 + e];
        for (int e = 0; e < 4; e++) pose[3 + e] = qq[e];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float* px = x + ((size_t)b * C + c) * T + t;
        const float xv = *px;
        float other = xv;                                          // body channels: x_ = body_pred
        if (c >= 3 * Jn && c < 3 * Jn + 3 * Np) {
            const int p = (c - 3 * Jn) / 3, ax = (c - 3 * Jn) % 3;
            const float* zp = zero_pose + ((size_t)b * Np + p) * 3;
            other = (R[ax * 3] * zp[0] + R[ax * 3 + 1] * zp[1] + R[ax * 3 + 2] * zp[2]) + pose[ax];
        } else if (c >= 3 * Jn + 3 * Np) {
            other = pose[c - 3 * Jn - 3 * Np];
        }
        *px = __fadd_rn(__fmul_rn(a, xv), __fmul_rn(a1, other));
    }
}
}  // namespace

/* ObjProjector.sample of the skeleton net: obj_quat (T,B,4) xyzw, obj_trans (T,B,3), joints (T,B,n_joints,3)
   -> quat_out (T,B,4) xyzw, trans_out (T,B,3) */
extern "C" int idb_projector_sample_skeleton(idb_handle* h, int T, int B, const float* obj_quat, const float* obj_trans, const float* joints,
                                             float* quat_out, float* trans_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !obj_quat || !obj_trans || !joints || !quat_out || !trans_out || T <= 0 || B <= 0) return IDB_ERR_ARG;
    if (!h->proj || h->proj->variant != 1) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init_skeleton first");
    Projector& p = *h->proj;
    cudaStream_t st = (cudaStream_t)stream;
    const int F = T * B;
    if (F > p.skel_cap) {
        h->epoch++;
        if (p.skel_ws) cudaFree(p.skel_ws);
        CUDA_TRY(h, cudaMalloc((void**)&p.skel_ws, sizeof(float) * (size_t)F * (6 + 9)));
        p.skel_cap = F;
    }
    float* ang6 = p.skel_ws; float* res = ang6 + (size_t)F * 6;
    k_quat_to_6d<<<(F + 127) / 128, 128, 0, st>>>(obj_quat, ang6, F);
    LAUNCH_CHECK(h);
    int rc = projector_run(h, T, B, ang6, obj_trans, joints, nullptr, res, st);
    if (rc) return rc;
    k_proj_to_quat<<<(F + 127) / 128, 128, 0, st>>>(res, quat_out, trans_out, F);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

/* denoised_fn of eval_skeleton.py:80-111 for an ACTIVE step, in place on x0 (B,1,C,T), C = 3 n_joints + 3 n_points + 7:
   the object pose of the inpainted motion goes through the skeleton correction net (conditioned on the predicted joints),
   the object keypoints are re-derived from the projected pose and zero_pose_obj (B,n_points,3), and
   x0 = (t/1000) x0 + (1 - t/1000) [body | keypoints | pose] for every sample.  (The reference also evaluates
   body_obj_to_contact (:96) but never uses its result.) */
extern "C" int idb_skeleton_correction_apply(idb_handle* h, int B, int T, int n_points, float* x0, const float* gt, const float* zero_pose_obj,
                                             int t, void* stream) {
    IDB_ENTER(h);
    if (!h || !x0 || !gt || !zero_pose_obj || B <= 0 || T <= 0 || n_points <= 0) return IDB_ERR_ARG;
    if (!h->proj || h->proj->variant != 1) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init_skeleton first");
    Projector& p = *h->proj;
    cudaStream_t st = (cudaStream_t)stream;
    const int F = T * B, Jn = p.P, C = 3 * Jn + 3 * n_points + 7;
    if (F > p.skel_hook_cap) {
        h->epoch++;
        if (p.skel_hook_ws) cudaFree(p.skel_hook_ws);
        CUDA_TRY(h, cudaMalloc((void**)&p.skel_hook_ws, sizeof(float) * (size_t)F * (Jn * 3 + 3 + 4 + 4 + 3)));
        p.skel_hook_cap = F;
    }
    float* joints = p.skel_hook_ws; float* gtr = joints + (size_t)F * Jn * 3; float* gq = gtr + (size_t)F * 3;
    float* pq = gq + (size_t)F * 4; float* ptr = pq + (size_t)F * 4;
    k_skel_gather<<<F, 64, 0, st>>>(x0, joints, gt, gtr, gq, B, T, C, Jn);
    LAUNCH_CHECK(h);
    int rc = idb_projector_sample_skeleton(h, T, B, gq, gtr, joints, pq, ptr, stream);
    if (rc) return rc;
    k_skel_blend<<<F, 128, 0, st>>>(x0, pq, ptr, zero_pose_obj, (float)t / 1000.0f, B, T, C, Jn, n_points);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

/* Debug / parity hook: device buffers cond_log [capacity][B] uint8 and contact_log [capacity][B][P] int32 that receive the
   decisions (condition, contact) of every correction step ENQUEUED from now on, in order (slot = running count, reset by
   this call; NULL switches the log off).  A captured whole-loop graph keeps writing the slots it was captured with. */
extern "C" int idb_correction_set_log(idb_handle* h, uint8_t* cond_log, int32_t* contact_log, int capacity) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    if (!h->proj) return idb_fail(h, IDB_ERR_STATE, "idb_projector_init first");
    if ((cond_log == nullptr) != (contact_log == nullptr) || capacity < 0) return IDB_ERR_ARG;
    Projector& p = *h->proj;
    p.log_cond = cond_log; p.log_contact = contact_log; p.log_cap = cond_log ? capacity : 0; p.log_n = 0;
    h->epoch++;      // captured graphs contain (or lack) the log copies
    return IDB_OK;
}

extern "C" int idb_correction_apply(idb_handle* h, float* x0, const float* gt, int t, uint8_t* condition_out,
                                    int32_t* contact_out, float* markers_out, float* o2h_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !x0 || !gt) return IDB_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = idb_correction_apply_dev(h, x0, gt, t, st);
    if (rc) return rc;
    Projector& p = *h->proj;
    const int F = p.cT * p.B;
    if (condition_out) CUDA_TRY(h, cudaMemcpyAsync(condition_out, p.cond, p.B, cudaMemcpyDefault, st));
    if (contact_out) CUDA_TRY(h, cudaMemcpyAsync(contact_out, p.contact, (size_t)p.B * p.P * 4, cudaMemcpyDefault, st));
    if (markers_out) CUDA_TRY(h, cudaMemcpyAsync(markers_out, p.markers, (size_t)F * p.P * 3 * 4, cudaMemcpyDefault, st));
    if (o2h_out) CUDA_TRY(h, cudaMemcpyAsync(o2h_out, p.o2h, (size_t)F * p.n_obj * 4, cudaMemcpyDefault, st));
    return IDB_OK;
}
