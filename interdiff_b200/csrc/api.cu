// Handle lifecycle of the C ABI (include/interdiff_b200.h).
#include "common.cuh"

void idb_denoiser_release(idb_handle* h);
void idb_sampler_release(idb_handle* h);
void idb_body_release(idb_handle* h);
void idb_projector_release(idb_handle* h);
int idb_denoiser_prepare_kernels(idb_handle* h);
void idb_sampler_drop_graphs(idb_handle* h);

extern "C" int idb_version(void) { return 100; }

extern "C" int idb_create(idb_handle** out) {
    if (!out) return IDB_ERR_ARG;
    *out = nullptr;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return IDB_ERR_CUDA;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return IDB_ERR_CUDA;
    idb_handle* h = new idb_handle();
    h->device = dev;
    h->sm_count = prop.multiProcessorCount;
    if (prop.major != 9) {
        // sm_90a-only library: refuse loudly rather than fall back
        h->err = "interdiff_b200 needs a Hopper (sm_90) device";
        *out = h;
        return IDB_ERR_CUDA;
    }
    int rc = idb_denoiser_prepare_kernels(h);
    *out = h;
    return rc;
}

extern "C" int idb_destroy(idb_handle* h) {
    IDB_ENTER(h);
    if (!h) return IDB_OK;
    idb_sampler_release(h);
    idb_denoiser_release(h);
    idb_projector_release(h);
    idb_body_release(h);
    if (h->scratch) cudaFree(h->scratch);
    if (h->metrics_ws) cudaFree(h->metrics_ws);
    delete h;
    return IDB_OK;
}

extern "C" const char* idb_last_error(const idb_handle* h) { return h ? h->err.c_str() : "null handle"; }
extern "C" long long idb_launch_count(const idb_handle* h) { return h ? h->launches : 0; }
extern "C" int idb_set_gemm_backend(idb_handle* h, int backend) {
    IDB_ENTER(h);
    if (!h || backend < 0 || backend > 1) return IDB_ERR_ARG;
    h->gemm_backend = backend;
    idb_sampler_drop_graphs(h);      // the captured step graphs contain the other backend's kernels
    return IDB_OK;
}

// Programmatic dependent launch between the kernels of a step (default on).  Changing it drops the
// captured step graphs so the next idb_p_sample_loop re-captures with the new launch attributes.
extern "C" int idb_set_dependent_launch(idb_handle* h, int on) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    h->pdl = on ? 1 : 0;
    idb_sampler_drop_graphs(h);
    return IDB_OK;
}

extern "C" int idb_set_nn_pruning(idb_handle* h, int on) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    h->nn_pruning = on ? 1 : 0;
    idb_sampler_drop_graphs(h);
    return IDB_OK;
}
/* test / bisecting hook: 0 = the SMPL-H blend GEMM without the multicast row-tile pairs (identical results) */
extern "C" int idb_debug_set_gemm_multicast(idb_handle* h, int on) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    h->gemm_multicast = on ? 1 : 0;
    idb_sampler_drop_graphs(h);
    return IDB_OK;
}
extern "C" double idb_debug_last_ms(const idb_handle* h) { return h ? h->last_ms : 0.0; }
extern "C" int idb_set_fused_mlp(idb_handle* h, int on) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    if (on == 10 || on == 11) h->fuse_attn = on - 10;     /* standard layers: attention halves in one launch */
    else if (on == 0 || on == 2) h->fused_mlp = on / 2;   /* 0 = two GEMMs, 2 = cluster kernel incl. the layer's final norm */
    else return idb_fail(h, IDB_ERR_ARG, "idb_set_fused_mlp: %d is not one of 0, 2, 10, 11", on);
    idb_sampler_drop_graphs(h);
    return IDB_OK;
}

extern long long* g_idb_gemm_trace;
/* test hook: out[M][256] = gelu(x w1^T + b1) w2^T + b2 + res through the fused cluster kernel (fp32 device inputs,
   x [M][256], w1 [1024][256], w2 [256][1024]); operands are split into fp16 pairs in temporary buffers.  out_hi / out_lo
   (NULL = none): the output's fp16 (hi, lo) pairs, row stride 256 like out.  Only rows < M of the outputs are written. */
extern "C" int idb_debug_mlp(idb_handle* h, const float* x, const float* w1, const float* b1, const float* w2, const float* b2,
                             const float* res, float* out, int M, int iters, long long* trace, const float* ln_w, const float* ln_b,
                             void* out_hi, void* out_lo, void* stream) {
    IDB_ENTER(h);
    if (!h || !x || !w1 || !b1 || !w2 || !b2 || !res || !out || M <= 0 || (out_hi == nullptr) != (out_lo == nullptr)) return IDB_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int Dm = 256, F = 1024;
    __half* buf = nullptr;
    const size_t nx = (size_t)M * Dm, nw = (size_t)F * Dm;
    CUDA_TRY(h, cudaMalloc((void**)&buf, sizeof(__half) * 2 * (nx + 2 * nw)));
    __half *xh = buf, *xl = xh + nx, *w1h = xl + nx, *w1l = w1h + nw, *w2h = w1l + nw, *w2l = w2h + nw;
    int rc = idb_split_tensor(h, x, Dm, xh, xl, Dm, M, Dm, st);
    if (!rc) rc = idb_split_tensor(h, w1, Dm, w1h, w1l, Dm, F, Dm, st);
    if (!rc) rc = idb_split_tensor(h, w2, F, w2h, w2l, F, Dm, F, st);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int i = 0; i < (iters > 0 ? iters : 1) && !rc; i++) {
        if (i == 0 && trace) g_idb_gemm_trace = trace;
        if (i == 1) cudaEventRecord(e0, st);
        rc = idb_mlp_wgmma(h, xh, xl, w1h, w1l, b1, w2h, w2l, b2, res, Dm, out, Dm, M, 0, st, ln_w, ln_b, (__half*)out_hi, (__half*)out_lo);
    }
    g_idb_gemm_trace = nullptr;
    cudaEventRecord(e1, st);
    cudaStreamSynchronize(st);
    if (iters > 1 && !rc) { float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1); h->last_ms = ms / (iters - 1); }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(buf);
    return rc;
}

/* test hook: one GEMM with every GemmArgs field a library caller sets (the tensor path's split-K onto a C the caller zeroed,
   the aux-zero side job, fp16 (hi, lo) operands and outputs, strides, single accumulator, dependent launch) */
extern "C" int idb_debug_gemm_ex(idb_handle* h, const idb_gemm_desc* d, void* stream) {
    IDB_ENTER(h);
    if (!h || !d) return IDB_ERR_ARG;
    GemmArgs g;
    g.A = d->A; g.A_hi = (const __half*)d->A_hi; g.A_lo = (const __half*)d->A_lo; g.lda = d->lda;
    g.W = d->W; g.W_hi = (const __half*)d->W_hi; g.W_lo = (const __half*)d->W_lo; g.ldw = d->ldw;
    g.bias = d->bias; g.res = d->res; g.ldr = d->ldr;
    g.C = d->C; g.C_hi = (__half*)d->C_hi; g.C_lo = (__half*)d->C_lo; g.ldc = d->ldc;
    g.M = d->M; g.N = d->N; g.K = d->K; g.epi = d->epi;
    g.ksplit = d->ksplit; g.zero = d->zero; g.zero_ld = d->zero_ld; g.zero_cols = d->zero_cols;
    g.pdl = d->pdl; g.single_acc = d->single_acc;
    g_idb_gemm_trace = d->trace;
    const int rc = idb_gemm_ex(h, g, (cudaStream_t)stream);
    g_idb_gemm_trace = nullptr;     // not consumed when the call took the SIMT path or failed before the launch
    return rc;
}

/* same GEMM launched `iters` times back to back from C (keeps host overhead per launch small) */
extern "C" int idb_debug_gemm_repeat(idb_handle* h, const float* A, const float* W, const float* bias, const float* res, float* C,
                                     int M, int N, int K, int epi, int iters, void* stream) {
    IDB_ENTER(h);
    if (!h || !A || !W || !C) return IDB_ERR_ARG;
    for (int i = 0; i < iters; i++) {
        int rc = idb_gemm(h, A, K, W, K, bias, res, N, C, N, M, N, K, epi, (cudaStream_t)stream);
        if (rc) return rc;
    }
    return IDB_OK;
}

static int g_idb_trace_epi = 0;
int idb_chain_set_gemm(unsigned long long* buf);
int idb_chain_set_denoiser(unsigned long long* buf);
/* chain timeline probe: buf = 64 lanes x (2 + 2 * capacity) uint64 (lane[0] = 0, lane[1] = capacity), NULL = off */
extern "C" int idb_debug_chain_trace(idb_handle* h, unsigned long long* buf) {
    IDB_ENTER(h);
    if (!h) return IDB_ERR_ARG;
    return (idb_chain_set_gemm(buf) | idb_chain_set_denoiser(buf)) ? IDB_ERR_CUDA : IDB_OK;
}
extern int g_idb_gemm_promote;
extern int g_idb_gemm_wide_tiles;
extern int g_idb_gemm_persistent;
/* test hook: k-blocks the big x big products accumulate in the tensor core between fp32 promotions (0 = default); 900 / 901: 128-column tiles off / on;
   910 / 911: one tile per CTA / the persistent schedule (default) of the 64-column kernel */
extern "C" int idb_debug_set_gemm_accumulators(int n) {
    if (n == 900 || n == 901) { g_idb_gemm_wide_tiles = n - 900; return IDB_OK; }
    if (n == 910 || n == 911) { g_idb_gemm_persistent = n - 910; return IDB_OK; }
    if (n >= 1000) { g_idb_trace_epi = n - 1000; return IDB_OK; }   // >= 1000: epi flags for idb_debug_gemm_presplit
    g_idb_gemm_promote = n;
    return IDB_OK;
}

/* x[rows][cols] -> fp16 (hi, lo) pairs with row stride ld_dst (device pointers) */
extern "C" int idb_debug_split(idb_handle* h, const float* x, void* hi, void* lo, int rows, int cols, int ld_dst, void* stream) {
    IDB_ENTER(h);
    if (!h || !x || !hi || !lo || rows <= 0 || cols <= 0 || ld_dst < cols) return IDB_ERR_ARG;
    return idb_split_tensor(h, x, cols, (__half*)hi, (__half*)lo, ld_dst, rows, cols, (cudaStream_t)stream);
}
/* GEMM on fp16 (hi, lo) operand pairs, `iters` launches; the first launch records the pipeline timeline when trace != NULL */
extern "C" int idb_debug_gemm_presplit(idb_handle* h, const void* A_hi, const void* A_lo, const void* W_hi, const void* W_lo,
                                       const float* bias, float* C, int M, int N, int K, int epi, int iters, long long* trace,
                                       void* stream) {
    IDB_ENTER(h);
    if (!h || !A_hi || !A_lo || !W_hi || !W_lo || !C) return IDB_ERR_ARG;
    GemmArgs g;
    g.A_hi = (const __half*)A_hi; g.A_lo = (const __half*)A_lo; g.lda = K; g.W_hi = (const __half*)W_hi; g.W_lo = (const __half*)W_lo; g.ldw = K;
    g.bias = bias; g.C = C; g.ldc = N; g.M = M; g.N = N; g.K = K; g.epi = (epi & ~128) | g_idb_trace_epi;
    if (epi & 128) g.ksplit = 2;   /* timing only: C is not re-zeroed between launches */
    for (int i = 0; i < iters; i++) {
        if (i == 0 && trace) g_idb_gemm_trace = trace;
        int rc = idb_gemm_ex(h, g, (cudaStream_t)stream);
        if (rc) return rc;
    }
    return IDB_OK;
}
