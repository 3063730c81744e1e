// Diffusion process: ancestral DDPM and DDIM sampling (START_X, FIXED_SMALL) around the denoiser.
// Replaces reference diffusion/gaussian_diffusion.py:160-197 (coefficient tables, float64 on the
// host exactly like the reference, then .float()), :253-275, :277-388, :496-548, :598-736, the DDIM
// sampler :738-788 and :885-999, and diffusion/respace.py:64-129.
//
// Every per-step scalar lives in a device table indexed by a device-side step counter, so one
// captured CUDA graph of a step can be replayed for every timestep without host patching.  The
// counter is moved by the last kernel of a step (k_step_io, denoiser.cu), which also prepares the
// next step's decoder input, so a plain step is: decoder body (GEMMs + attention) + one tail kernel.
// DDPM and DDIM differ only in the table: both updates are c1[i] x0 + c2[i] x_t + sigma_nz[i] eps.
#include "common.cuh"

int idb_denoiser_tokens(idb_handle* h, const float* x, const long long* tstep, cudaStream_t st);
int idb_denoiser_body(idb_handle* h, cudaStream_t st);
int idb_denoiser_heads(idb_handle* h, const float* gt, const unsigned char* mask, float* out, cudaStream_t st);
// i_host >= 0: the step index is known when the launch is enqueued (plain launches, whole-loop graph); -1: device counter.
// noise null: no eps term; clip: x0 clamped to [-1, 1] before the update
int idb_step_finish(idb_handle* h, const float* x0, const float* xt, const float* noise, int tape_mode, float* x_next, int emit_next,
                    cudaStream_t st, int i_host, int clip);
int idb_step_tail(idb_handle* h, const float* gt, const unsigned char* mask, float* x0_out, const float* xt, const float* noise,
                  int tape_mode, float* x_next, int emit_next, cudaStream_t st, int i_host, int clip);
int idb_correction_apply_dev(idb_handle* h, float* x0, const float* gt, int t, cudaStream_t st);
int idb_correction_prepare(idb_handle* h, int B, int T);

struct Sampler {
    float *x_a = nullptr, *x0 = nullptr;
    size_t numel = 0;
    // graph-stable copies of the caller's inpainting tensors and a device slot holding the caller's tape pointer:
    // the captured graphs only reference buffers owned by the handle, so a new tape / gt / mask tensor per call
    // does not force a re-capture
    float* gt_buf = nullptr; unsigned char* mask_buf = nullptr; const float** tape_slot = nullptr;
    cudaGraphExec_t step_graph = nullptr;     // predict + finish for a plain step
    cudaGraphExec_t predict_graph = nullptr;  // predict only (correction steps)
    cudaGraphExec_t loop_graph = nullptr;     // the whole loop (use_graph == 2)
    // what the cached graphs were captured for; `epoch` = idb_handle::epoch at capture (bumped by every call that
    // frees / reallocates / re-routes anything a captured node points at)
    int gB = 0, gT = 0, g_mask = -1, g_tape = -1, g_clip = -1; long long g_epoch = -1;
    int lB = 0, lT = 0, l_mask = -1, l_n = 0, l_corr = -1, l_tape = -1, l_clip = -1; long long l_epoch = -1;
    int launches_per_step = 0, launches_per_predict = 0; long long launches_per_loop = 0;
};

namespace {

__global__ void k_set_counter(int* counter, int v) { *counter = v; }
__global__ void k_loop_begin(int* counter, int v, const float** slot, const float* tape) { *counter = v; *slot = tape; }

void drop_graphs(Sampler& s) {
    if (s.step_graph) { cudaGraphExecDestroy(s.step_graph); s.step_graph = nullptr; }
    if (s.predict_graph) { cudaGraphExecDestroy(s.predict_graph); s.predict_graph = nullptr; }
    if (s.loop_graph) { cudaGraphExecDestroy(s.loop_graph); s.loop_graph = nullptr; }
}

}  // namespace

// upload a finished step table; every captured graph is dropped (they point at the old table and were captured for the
// other table kind)
static int load_table(idb_handle* h, const std::vector<StepParams>& tab, int kind) {
    Diffusion& df = h->diff;
    const int n = (int)tab.size();
    if (df.tbl) { cudaFree(df.tbl); df.tbl = nullptr; df.n = 0; }
    h->epoch++;
    if (h->sampler) drop_graphs(*h->sampler);
    CUDA_TRY(h, cudaMalloc((void**)&df.tbl, sizeof(StepParams) * n));
    CUDA_TRY(h, cudaMemcpy(df.tbl, tab.data(), sizeof(StepParams) * n, cudaMemcpyHostToDevice));
    df.host = tab;
    df.n = n;
    df.kind = kind;
    df.noisy = false;
    for (const StepParams& p : tab) df.noisy |= p.sigma_nz != 0.0f;
    return IDB_OK;
}

extern "C" int idb_diffusion_init(idb_handle* h, const double* betas, const int64_t* timestep_map, int n) {
    IDB_ENTER(h);
    if (!h || !betas || n <= 0) return IDB_ERR_ARG;
    // float64 tables exactly as GaussianDiffusion.__init__ (gaussian_diffusion.py:160-197)
    std::vector<double> ac(n), ac_prev(n), post_var(n), logvar(n), c1(n), c2(n);
    double prod = 1.0;
    for (int i = 0; i < n; i++) {
        if (!(betas[i] > 0 && betas[i] <= 1)) return idb_fail(h, IDB_ERR_ARG, "betas must be in (0,1]");
        prod *= (1.0 - betas[i]);
        ac[i] = prod;
        ac_prev[i] = i == 0 ? 1.0 : ac[i - 1];
    }
    for (int i = 0; i < n; i++) {
        post_var[i] = betas[i] * (1.0 - ac_prev[i]) / (1.0 - ac[i]);
        c1[i] = betas[i] * std::sqrt(ac_prev[i]) / (1.0 - ac[i]);
        c2[i] = (1.0 - ac_prev[i]) * std::sqrt(1.0 - betas[i]) / (1.0 - ac[i]);
    }
    for (int i = 0; i < n; i++) logvar[i] = std::log(i == 0 ? post_var[n > 1 ? 1 : 0] : post_var[i]);
    std::vector<StepParams> tab(n);
    for (int i = 0; i < n; i++) {
        StepParams& p = tab[i];
        p.t = timestep_map ? (long long)timestep_map[i] : i;
        p.c1 = (float)c1[i];
        p.c2 = (float)c2[i];
        // reference: th.exp(0.5 * float32(logvar)) evaluated in float32
        const float lv = (float)logvar[i];
        p.sigma_nz = i == 0 ? 0.0f : expf(0.5f * lv);
        p.pad = 0.f;
    }
    return load_table(h, tab, DIFF_DDPM);
}

// DDIM (gaussian_diffusion.py:738-788) for START_X: with eps = (sqrt_recip_ac x_t - x0) / sqrt_recipm1_ac (:407-411),
//   x_prev = sqrt(ac_prev) x0 + k eps + 1[i != 0] sigma noise,  k = sqrt(1 - ac_prev - sigma^2),
//   sigma = eta sqrt((1 - ac_prev) / (1 - ac)) sqrt(1 - ac / ac_prev)
// is  a x0 + b x_t + sigma_nz noise  with  a = sqrt(ac_prev) - k / sqrt_recipm1_ac,  b = k sqrt_recip_ac / sqrt_recipm1_ac.
// Folded in float64 and rounded once, so the float32 cancellation in `a` that the reference's own evaluation carries is
// absent; at i = 0 (ac_prev = 1) a = 1, b = 0, sigma = 0 exactly, so the final sample is x0.
extern "C" int idb_diffusion_init_ddim(idb_handle* h, const double* betas, const int64_t* timestep_map, int n, double eta) {
    IDB_ENTER(h);
    if (!h || !betas || n <= 0) return IDB_ERR_ARG;
    if (!(eta >= 0.0) || !std::isfinite(eta)) return idb_fail(h, IDB_ERR_ARG, "eta must be finite and >= 0");
    std::vector<StepParams> tab(n);
    double ac = 1.0;
    for (int i = 0; i < n; i++) {
        if (!(betas[i] > 0 && betas[i] <= 1)) return idb_fail(h, IDB_ERR_ARG, "betas must be in (0,1]");
        const double ac_prev = ac;
        ac *= (1.0 - betas[i]);
        const double sqrt_recip = std::sqrt(1.0 / ac), sqrt_recipm1 = std::sqrt(1.0 / ac - 1.0);
        const double sigma = eta * std::sqrt((1.0 - ac_prev) / (1.0 - ac)) * std::sqrt(1.0 - ac / ac_prev);
        const double k2 = 1.0 - ac_prev - sigma * sigma;
        if (!(k2 >= 0.0))
            return idb_fail(h, IDB_ERR_ARG, "eta %g gives 1 - alpha_bar_prev - sigma^2 < 0 at step %d (the reference would produce NaN)", eta, i);
        const double k = std::sqrt(k2);
        StepParams& p = tab[i];
        p.t = timestep_map ? (long long)timestep_map[i] : i;
        p.c1 = (float)(std::sqrt(ac_prev) - k / sqrt_recipm1);
        p.c2 = (float)(k * sqrt_recip / sqrt_recipm1);
        p.sigma_nz = i == 0 ? 0.0f : (float)sigma;
        p.pad = 0.f;
    }
    return load_table(h, tab, DIFF_DDIM);
}

static int sampler_ready(idb_handle* h, size_t numel) {
    if (!h->diff.n) return idb_fail(h, IDB_ERR_STATE, "idb_diffusion_init first");
    if (!h->den.B) return idb_fail(h, IDB_ERR_STATE, "idb_denoiser_bind first");
    if (!h->sampler) h->sampler = new Sampler();
    Sampler& s = *h->sampler;
    if (s.numel != numel) {
        drop_graphs(s);
        if (s.x_a) { cudaFree(s.x_a); cudaFree(s.x0); cudaFree(s.gt_buf); cudaFree(s.mask_buf); s.x_a = nullptr; }
        CUDA_TRY(h, cudaMalloc((void**)&s.x_a, numel * sizeof(float)));
        CUDA_TRY(h, cudaMalloc((void**)&s.x0, numel * sizeof(float)));
        CUDA_TRY(h, cudaMalloc((void**)&s.gt_buf, numel * sizeof(float)));
        CUDA_TRY(h, cudaMalloc((void**)&s.mask_buf, numel));
        if (!s.tape_slot) CUDA_TRY(h, cudaMalloc((void**)&s.tape_slot, sizeof(float*)));
        s.numel = numel;
    }
    return IDB_OK;
}

static size_t sample_numel(idb_handle* h) {
    const idb_denoiser_config& c = h->den.cfg;
    return (size_t)h->den.B * (c.c_body + c.c_obj + c.c_extra) * h->den.T;
}

// predict with the device counter already set: tokens from x_t, decoder, heads
static int predict_dev(idb_handle* h, const float* x_t, const float* gt, const unsigned char* mask, float* x0, cudaStream_t st) {
    int rc;
    if ((rc = idb_denoiser_tokens(h, x_t, nullptr, st))) return rc;
    if ((rc = idb_denoiser_body(h, st))) return rc;
    return idb_denoiser_heads(h, gt, mask, x0, st);
}

static int set_step(idb_handle* h, int i, cudaStream_t st) {
    if (!h->den.step_cur) return idb_fail(h, IDB_ERR_STATE, "idb_denoiser_bind first");
    k_set_counter<<<1, 1, 0, st>>>(h->den.step_cur, i);
    LAUNCH_CHECK(h);
    return IDB_OK;
}

extern "C" int idb_p_sample_predict(idb_handle* h, int i, const float* x_t, const float* gt, const uint8_t* mask, float* x0_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !x_t || !x0_out) return IDB_ERR_ARG;
    if (i < 0 || i >= h->diff.n) return idb_fail(h, IDB_ERR_ARG, "step index out of range");
    if ((gt == nullptr) != (mask == nullptr)) return idb_fail(h, IDB_ERR_ARG, "gt and mask must be given together");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = set_step(h, i, st);
    if (rc) return rc;
    return predict_dev(h, x_t, gt, mask, x0_out, st);
}

extern "C" int idb_p_sample_finish(idb_handle* h, int i, const float* x0, const float* x_t, const float* noise, float* x_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !x0 || !x_t || !noise || !x_out) return IDB_ERR_ARG;
    if (i < 0 || i >= h->diff.n) return idb_fail(h, IDB_ERR_ARG, "step index out of range");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = set_step(h, i, st);
    if (rc) return rc;
    return idb_step_finish(h, x0, x_t, noise, 0, x_out, 0, st, -1, 0);
}

extern "C" int idb_p_sample(idb_handle* h, int i, const float* x_t, const float* noise, const float* gt, const uint8_t* mask,
                            float* x_out, float* x0_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !x_t || !noise || !x_out) return IDB_ERR_ARG;
    if (i < 0 || i >= h->diff.n) return idb_fail(h, IDB_ERR_ARG, "step index out of range");
    if ((gt == nullptr) != (mask == nullptr)) return idb_fail(h, IDB_ERR_ARG, "gt and mask must be given together");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = set_step(h, i, st);
    if (rc) return rc;
    if ((rc = idb_denoiser_tokens(h, x_t, nullptr, st))) return rc;
    if ((rc = idb_denoiser_body(h, st))) return rc;
    return idb_step_tail(h, gt, mask, x0_out, x_t, noise, 0, x_out, 0, st, i, 0);
}

// One plain step / one correction step on the sampler's own buffers (x in place in s.x_a; gt / mask = the
// graph-stable copies; noise through the tape slot, or none: `noise` is s.tape_slot or null).
static int plain_step(idb_handle* h, Sampler& s, const float* gt, const unsigned char* mask, const float* noise, int clip,
                      cudaStream_t st, int i_host) {
    int rc = idb_denoiser_body(h, st);
    if (rc) return rc;
    return idb_step_tail(h, gt, mask, nullptr, s.x_a, noise, 2, s.x_a, 1, st, i_host, clip);
}
static int predict_part(idb_handle* h, Sampler& s, const float* gt, const unsigned char* mask, cudaStream_t st) {
    int rc = idb_denoiser_body(h, st);
    if (rc) return rc;
    return idb_denoiser_heads(h, gt, mask, s.x0, st);
}
// reference order inside p_mean_variance (gaussian_diffusion.py:305-376): model -> inpaint blend -> denoised_fn -> clip ->
// update; there is NO re-inpainting after the hook.  The hook receives the UN-mapped step index i (:356).
// i_host: i when every step of the loop is enqueued with its index (plain launches, whole-loop graph), -1 when the other steps
// replay a captured graph that reads - and therefore needs this step to move - the device counter
static int correction_tail(idb_handle* h, Sampler& s, const float* gt, const float* noise, int clip, int i, cudaStream_t st, int i_host) {
    int rc = idb_correction_apply_dev(h, s.x0, gt, i, st);
    if (rc) return rc;
    return idb_step_finish(h, s.x0, s.x_a, noise, 2, s.x_a, 1, st, i_host, clip);
}
static inline bool correction_gate(int correction, int i) { return correction && i <= 500 && (i % 50 == 0); }   // eval_smpl_short.py:86-88

template <typename Body>
static int capture_graph(idb_handle* h, cudaGraphExec_t* out, long long* n_launches, Body&& body) {
    cudaStream_t cs;
    CUDA_TRY(h, cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    cudaGraph_t g = nullptr;
    const long long saved = h->launches;
    cudaError_t ce = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) { cudaStreamDestroy(cs); return idb_fail(h, IDB_ERR_CUDA, "graph capture failed to start: %s", cudaGetErrorString(ce)); }
    int rc = body(cs);
    ce = cudaStreamEndCapture(cs, &g);
    *n_launches = h->launches - saved;
    h->launches = saved;
    if (rc || ce != cudaSuccess) {
        if (g) cudaGraphDestroy(g);
        cudaStreamDestroy(cs);
        return rc ? rc : idb_fail(h, IDB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
    }
    ce = cudaGraphInstantiate(out, g, 0);
    cudaGraphDestroy(g);
    cudaStreamDestroy(cs);
    if (ce != cudaSuccess) return idb_fail(h, IDB_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
    return IDB_OK;
}

// The loop of idb_p_sample_loop and idb_ddim_sample_loop over the loaded table: x starts as x_T; tape (n + 1 entries, entry
// k + 1 = eps of the k-th executed step) or null = no noise term.
// use_graph: 0 = plain launches, 1 = one captured graph per step (replayed n times), 2 = the whole loop as one graph.
static int run_loop(idb_handle* h, const float* x_T, const float* tape, const float* gt, const uint8_t* mask, int correction, int clip,
                    int use_graph, float* x_out, cudaStream_t st) {
    if ((gt == nullptr) != (mask == nullptr)) return idb_fail(h, IDB_ERR_ARG, "gt and mask must be given together");
    if (correction && !gt) return idb_fail(h, IDB_ERR_ARG, "the correction hook reads the inpainted ground truth (eval_smpl_short.py:113): gt required");
    const size_t numel = sample_numel(h);
    int rc = sampler_ready(h, numel);
    if (rc) return rc;
    Sampler& s = *h->sampler;
    Diffusion& df = h->diff;
    const int n = df.n, has_mask = gt ? 1 : 0, has_tape = tape ? 1 : 0;
    clip = clip ? 1 : 0;
    if (correction && (rc = idb_correction_prepare(h, h->den.B, h->den.T))) return rc;   // workspaces sized before anything is captured
    const float* g_gt = gt ? s.gt_buf : nullptr;
    const unsigned char* g_mask = gt ? s.mask_buf : nullptr;
    const float* g_noise = tape ? reinterpret_cast<const float*>(s.tape_slot) : nullptr;
    // x lives in s.x_a for the whole loop (the update is elementwise, so in place is safe; x0 is separate)
    CUDA_TRY(h, cudaMemcpyAsync(s.x_a, x_T, numel * sizeof(float), cudaMemcpyDefault, st));
    if (gt) {
        CUDA_TRY(h, cudaMemcpyAsync(s.gt_buf, gt, numel * sizeof(float), cudaMemcpyDefault, st));
        CUDA_TRY(h, cudaMemcpyAsync(s.mask_buf, mask, numel, cudaMemcpyDefault, st));
    }
    k_loop_begin<<<1, 1, 0, st>>>(h->den.step_cur, n - 1, s.tape_slot, tape);
    LAUNCH_CHECK(h);

    if (use_graph == 2) {
        if (!s.loop_graph || s.l_epoch != h->epoch || s.lB != h->den.B || s.lT != h->den.T || s.l_mask != has_mask || s.l_n != n ||
            s.l_corr != (correction ? 1 : 0) || s.l_tape != has_tape || s.l_clip != clip) {
            if (s.loop_graph) { cudaGraphExecDestroy(s.loop_graph); s.loop_graph = nullptr; }
            rc = capture_graph(h, &s.loop_graph, &s.launches_per_loop, [&](cudaStream_t cs) {
                int r = idb_denoiser_tokens(h, s.x_a, nullptr, cs);
                for (int i = n - 1; i >= 0 && !r; i--) {
                    if (!correction_gate(correction, i)) r = plain_step(h, s, g_gt, g_mask, g_noise, clip, cs, i);
                    else { r = predict_part(h, s, g_gt, g_mask, cs); if (!r) r = correction_tail(h, s, g_gt, g_noise, clip, i, cs, i); }
                }
                return r;
            });
            if (rc) return rc;
            s.l_epoch = h->epoch; s.lB = h->den.B; s.lT = h->den.T; s.l_mask = has_mask; s.l_n = n; s.l_corr = correction ? 1 : 0;
            s.l_tape = has_tape; s.l_clip = clip;
        }
        CUDA_TRY(h, cudaGraphLaunch(s.loop_graph, st));
        h->launches += s.launches_per_loop;
        CUDA_TRY(h, cudaMemcpyAsync(x_out, s.x_a, numel * sizeof(float), cudaMemcpyDefault, st));
        return IDB_OK;
    }

    // decoder input of the first step; every later step gets its tokens from the previous step's tail
    if ((rc = idb_denoiser_tokens(h, s.x_a, nullptr, st))) return rc;
    const bool graph_ok = use_graph != 0;
    if (graph_ok && (!s.step_graph || s.g_epoch != h->epoch || s.gB != h->den.B || s.gT != h->den.T || s.g_mask != has_mask ||
                     s.g_tape != has_tape || s.g_clip != clip)) {
        if (s.step_graph) { cudaGraphExecDestroy(s.step_graph); s.step_graph = nullptr; }
        if (s.predict_graph) { cudaGraphExecDestroy(s.predict_graph); s.predict_graph = nullptr; }
        long long nl = 0;
        if ((rc = capture_graph(h, &s.step_graph, &nl, [&](cudaStream_t cs) { return plain_step(h, s, g_gt, g_mask, g_noise, clip, cs, -1); })))
            return rc;
        s.launches_per_step = (int)nl;
        if ((rc = capture_graph(h, &s.predict_graph, &nl, [&](cudaStream_t cs) { return predict_part(h, s, g_gt, g_mask, cs); }))) return rc;
        s.launches_per_predict = (int)nl;
        s.g_epoch = h->epoch; s.gB = h->den.B; s.gT = h->den.T; s.g_mask = has_mask; s.g_tape = has_tape; s.g_clip = clip;
    }
    for (int i = n - 1; i >= 0; i--) {
        if (!correction_gate(correction, i)) {
            if (graph_ok) {
                CUDA_TRY(h, cudaGraphLaunch(s.step_graph, st));
                h->launches += s.launches_per_step;
            } else if ((rc = plain_step(h, s, g_gt, g_mask, g_noise, clip, st, i))) return rc;
        } else {
            if (graph_ok) {
                CUDA_TRY(h, cudaGraphLaunch(s.predict_graph, st));
                h->launches += s.launches_per_predict;
            } else if ((rc = predict_part(h, s, g_gt, g_mask, st))) return rc;
            if ((rc = correction_tail(h, s, g_gt, g_noise, clip, i, st, graph_ok ? -1 : i))) return rc;
        }
    }
    CUDA_TRY(h, cudaMemcpyAsync(x_out, s.x_a, numel * sizeof(float), cudaMemcpyDefault, st));
    return IDB_OK;
}

extern "C" int idb_p_sample_loop(idb_handle* h, const float* tape, const float* gt, const uint8_t* mask, int correction,
                                 int use_graph, float* x_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !tape || !x_out) return IDB_ERR_ARG;
    return run_loop(h, tape, tape, gt, mask, correction, 0, use_graph, x_out, (cudaStream_t)stream);
}

extern "C" int idb_ddim_sample_loop(idb_handle* h, const float* x_T, const float* tape, const float* gt, const uint8_t* mask,
                                    int correction, int clip_denoised, int use_graph, float* x_out, void* stream) {
    IDB_ENTER(h);
    if (!h || !x_T || !x_out) return IDB_ERR_ARG;
    if (!h->diff.n || h->diff.kind != DIFF_DDIM) return idb_fail(h, IDB_ERR_STATE, "idb_diffusion_init_ddim first (a DDPM table is loaded)");
    if (!tape && h->diff.noisy) return idb_fail(h, IDB_ERR_ARG, "eta > 0: the loop needs a noise tape");
    return run_loop(h, x_T, tape, gt, mask, correction, clip_denoised, use_graph, x_out, (cudaStream_t)stream);
}

void idb_sampler_drop_graphs(idb_handle* h) {
    h->epoch++;
    if (h->sampler) drop_graphs(*h->sampler);
}

void idb_sampler_release(idb_handle* h) {
    if (h->sampler) {
        Sampler& s = *h->sampler;
        drop_graphs(s);
        if (s.x_a) { cudaFree(s.x_a); cudaFree(s.x0); cudaFree(s.gt_buf); cudaFree(s.mask_buf); }
        if (s.tape_slot) cudaFree(s.tape_slot);
        delete h->sampler;
        h->sampler = nullptr;
    }
    if (h->diff.tbl) cudaFree(h->diff.tbl);
    h->diff = Diffusion();
}
