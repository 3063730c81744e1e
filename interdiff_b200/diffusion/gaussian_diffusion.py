"""Host-side mirror of reference diffusion/gaussian_diffusion.py for the SAMPLING path
(ancestral DDPM and DDIM; START_X / FIXED_SMALL as configured by model/diffusion_smpl.py:251-284).

Same public surface the callers use (SURVEY.md section 8b): get_named_beta_schedule,
ModelMeanType / ModelVarType / LossType, GaussianDiffusion.{q_sample, q_posterior_mean_variance,
p_mean_variance, p_sample, p_sample_loop, p_sample_loop_progressive, ddim_sample, ddim_sample_loop,
ddim_sample_loop_progressive, ddim_reverse_sample, training_losses (forward values), num_timesteps}.
PLMS and the VB terms are out of scope (never reached by the reference's scripts, SURVEY 2a #1) and raise
NotImplementedError.

When `model` is an interdiff_b200 MDM the work runs in libinterdiff_b200.so: the whole loop as
CUDA-graph replays when no Python hook is attached (or the hook is the fused correction), and
step-by-step around an arbitrary `denoised_fn` callback otherwise.  DDPM and DDIM share the engine's one step
table: the first call of the other sampler (or another DDIM eta) on an engine re-initialises the table (a few
microseconds of host work and one small upload) and the next whole loop re-captures its CUDA graph (a few
milliseconds) - alternate samplers on separate engines when that matters.
"""
import enum
import math

import numpy as np
import torch as th


def get_named_beta_schedule(schedule_name, num_diffusion_timesteps, scale_betas=1.0):
    """reference gaussian_diffusion.py:20-44"""
    n = num_diffusion_timesteps
    if schedule_name == "linear":
        scale = scale_betas * 1000 / n
        return np.linspace(scale * 0.0001, scale * 0.02, n, dtype=np.float64)
    if schedule_name == "cosine":
        return betas_for_alpha_bar(n, lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2)
    raise NotImplementedError(f"unknown beta schedule: {schedule_name}")


def betas_for_alpha_bar(num_diffusion_timesteps, alpha_bar, max_beta=0.999):
    """reference gaussian_diffusion.py:47-64"""
    n = num_diffusion_timesteps
    return np.array([min(1 - alpha_bar((i + 1) / n) / alpha_bar(i / n), max_beta) for i in range(n)])


class ModelMeanType(enum.Enum):
    PREVIOUS_X = enum.auto()
    START_X = enum.auto()
    EPSILON = enum.auto()


class ModelVarType(enum.Enum):
    LEARNED = enum.auto()
    FIXED_SMALL = enum.auto()
    FIXED_LARGE = enum.auto()
    LEARNED_RANGE = enum.auto()


class LossType(enum.Enum):
    MSE = enum.auto()
    RESCALED_MSE = enum.auto()
    KL = enum.auto()
    RESCALED_KL = enum.auto()

    def is_vb(self):
        return self in (LossType.KL, LossType.RESCALED_KL)


def _extract_into_tensor(arr, timesteps, broadcast_shape):
    """reference gaussian_diffusion.py:1611-1623"""
    res = th.from_numpy(arr).to(device=timesteps.device)[timesteps].float()
    while len(res.shape) < len(broadcast_shape):
        res = res[..., None]
    return res.expand(broadcast_shape)


class GaussianDiffusion:
    def __init__(self, *, betas, model_mean_type, model_var_type, loss_type, rescale_timesteps=False, lambda_vel=0.0, **_unused):
        if model_mean_type != ModelMeanType.START_X or model_var_type != ModelVarType.FIXED_SMALL:
            raise NotImplementedError("interdiff_b200 implements the reference's sampling configuration only: "
                                      "START_X mean, FIXED_SMALL variance (model/diffusion_smpl.py:266-284)")
        self.model_mean_type, self.model_var_type, self.loss_type = model_mean_type, model_var_type, loss_type
        self.rescale_timesteps, self.lambda_vel = rescale_timesteps, lambda_vel
        betas = np.array(betas, dtype=np.float64)
        assert betas.ndim == 1 and (betas > 0).all() and (betas <= 1).all()
        self.betas = betas
        self.num_timesteps = int(betas.shape[0])
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        self.alphas_cumprod_next = np.append(self.alphas_cumprod[1:], 0.0)
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.timestep_map = list(range(self.num_timesteps))  # SpacedDiffusion overrides

    # ---- closed-form pieces (cheap elementwise torch; not on the per-step device path)
    def q_sample(self, x_start, t, noise=None):
        if noise is None:
            noise = th.randn_like(x_start)
        return (_extract_into_tensor(self.sqrt_alphas_cumprod, t, x_start.shape) * x_start
                + _extract_into_tensor(self.sqrt_one_minus_alphas_cumprod, t, x_start.shape) * noise)

    def q_posterior_mean_variance(self, x_start, x_t, t):
        mean = (_extract_into_tensor(self.posterior_mean_coef1, t, x_t.shape) * x_start
                + _extract_into_tensor(self.posterior_mean_coef2, t, x_t.shape) * x_t)
        return (mean, _extract_into_tensor(self.posterior_variance, t, x_t.shape),
                _extract_into_tensor(self.posterior_log_variance_clipped, t, x_t.shape))

    def _scale_timesteps(self, t):
        return t

    # ---- engine plumbing
    def _prepare(self, model, model_kwargs, T=None, kind=("ddpm", None)):
        """Returns (engine, gt, mask): binds cond, makes sure the tables live in the model's engine.  T = number of
        frames of the sample (x.shape[-1] / shape[-1]): the inpainting keys are optional upstream (:307).
        kind: the step table the caller needs, ("ddpm", None) or ("ddim", eta); None = any of this schedule (the
        caller only runs the model, whose timesteps both kinds share)."""
        if not hasattr(model, "engine_for"):
            raise TypeError("interdiff_b200 diffusion drives interdiff_b200 models only (no eager fallback)")
        y = (model_kwargs or {}).get("y")
        if y is None:
            raise KeyError("model_kwargs['y'] is required (gaussian_diffusion.py:307 dereferences it)")
        eng = model.engine_for(y["cond"].device)
        model.bind_kwargs(eng, model_kwargs, T=T)
        key = (id(eng), self.num_timesteps)
        if (getattr(self, "_eng_key", None) != key or eng.n_steps != self.num_timesteps or getattr(eng, "_diff_owner", None) is not self
                or (kind is not None and eng.diffusion_kind != kind)):
            if kind is not None and kind[0] == "ddim":
                eng.init_diffusion_ddim(self.betas, self.timestep_map, eta=kind[1])
            else:
                eng.init_diffusion(self.betas, self.timestep_map)
            eng._diff_owner = self
            self._eng_key = key
        gt, mask = y.get("inpainted_motion"), y.get("inpainting_mask")
        if (gt is None) != (mask is None):
            gt = mask = None
        return eng, gt, mask

    @staticmethod
    def _uniform_step(t):
        i = int(t[0])
        if not bool((t == i).all()):
            raise NotImplementedError("per-sample timesteps inside p_sample are not supported (the sampling loop uses a uniform t)")
        return i

    def p_mean_variance(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        eng, gt, mask = self._prepare(model, model_kwargs, T=x.shape[-1])
        i = self._uniform_step(t)
        x0 = eng.p_sample_predict(i, x, gt, mask)
        if denoised_fn is not None:
            x0 = denoised_fn(x0, t, model_kwargs)
        if clip_denoised:
            x0 = x0.clamp(-1, 1)
        mean, var, logvar = self.q_posterior_mean_variance(x0, x, t)
        return {"mean": mean, "variance": var, "log_variance": logvar, "pred_xstart": x0}

    def p_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None, const_noise=False,
                 _noise=None):
        if cond_fn is not None:
            raise NotImplementedError("cond_fn guidance is not on the reference's sampling path")
        eng, gt, mask = self._prepare(model, model_kwargs, T=x.shape[-1])
        i = self._uniform_step(t)
        x0 = eng.p_sample_predict(i, x, gt, mask)
        if denoised_fn is not None:
            x0 = denoised_fn(x0, t, model_kwargs)
        if clip_denoised:
            x0 = x0.clamp(-1, 1)
        noise = th.randn_like(x) if _noise is None else _noise     # _noise: this step's eps drawn up front by the loop
        if const_noise:
            noise = noise[[0]].repeat(x.shape[0], 1, 1, 1)
        return {"sample": eng.p_sample_finish(i, x0, x, noise), "pred_xstart": x0}

    def p_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                  model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                                  randomize_class=False, cond_fn_with_grad=False, const_noise=False):
        if cond_fn is not None or cond_fn_with_grad or randomize_class:
            raise NotImplementedError("classifier guidance options are not on the reference's sampling path")
        eng, gt, mask = self._prepare(model, model_kwargs, T=shape[-1])
        img = noise if noise is not None else th.randn(*shape, device=eng.device)
        if noise is None and gt is not None:
            img = (img * ~mask) + (gt * mask)   # initial inpaint blend (gaussian_diffusion.py:694-699)
        if skip_timesteps and init_image is None:
            init_image = th.zeros_like(img)
        indices = list(range(self.num_timesteps))[skip_timesteps:][::-1]
        if init_image is not None:
            img = self.q_sample(init_image, th.full((shape[0],), indices[0], device=eng.device, dtype=th.long), img)
        # every step's eps drawn up front in ONE generator call, exactly like the in-library loop (same seed -> the
        # callback path and the fused path see the same noise); the reference draws th.randn_like(x) per step (:532)
        from ..sampling import draw_tape
        tape = draw_tape(eng, img, len(indices))
        if progress:
            from tqdm.auto import tqdm
            indices = tqdm(indices)
        for k, i in enumerate(indices):
            t = th.full((shape[0],), i, device=eng.device, dtype=th.long)
            with th.no_grad():
                out = self.p_sample(model, img, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                    model_kwargs=model_kwargs, const_noise=const_noise, _noise=tape[k + 1])
            yield out
            img = out["sample"]

    def p_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                      device=None, progress=False, skip_timesteps=0, init_image=None, randomize_class=False,
                      cond_fn_with_grad=False, dump_steps=None, const_noise=False):
        fused_hook = denoised_fn is None or getattr(denoised_fn, "is_fused_correction", False)
        plain = (fused_hook and not clip_denoised and cond_fn is None and not progress and not skip_timesteps and init_image is None
                 and not randomize_class and dump_steps is None and not const_noise)
        if plain:
            # whole loop in the library: one CUDA-graph replay per step
            eng, gt, mask = self._prepare(model, model_kwargs, T=shape[-1])
            x_T = noise if noise is not None else th.randn(*shape, device=eng.device)
            if noise is None and gt is not None:
                x_T = (x_T * ~mask) + (gt * mask)
            from ..sampling import draw_tape
            tape = draw_tape(eng, x_T, self.num_timesteps)
            correction = denoised_fn is not None
            if correction:
                denoised_fn.bind(eng, model_kwargs)
            return eng.p_sample_loop(tape, gt, mask, correction=correction, use_graph=True)
        final, dump = None, []
        for k, sample in enumerate(self.p_sample_loop_progressive(
                model, shape, noise=noise, clip_denoised=clip_denoised, denoised_fn=denoised_fn, cond_fn=cond_fn,
                model_kwargs=model_kwargs, device=device, progress=progress, skip_timesteps=skip_timesteps,
                init_image=init_image, randomize_class=randomize_class, cond_fn_with_grad=cond_fn_with_grad, const_noise=const_noise)):
            if dump_steps is not None and k in dump_steps:
                dump.append(sample["sample"].clone())
            final = sample
        return dump if dump_steps is not None else final["sample"]

    def training_losses(self, model, x_start, t, model_kwargs=None, noise=None, dataset=None):
        """Reference gaussian_diffusion.py:1233-1368 for the shipped configuration (MSE loss, START_X, FIXED_SMALL): returns
        (model_output, target) exactly like upstream - x_t = q_sample(x_start, t, noise), the inpainting blend (:1264-1268),
        one denoiser forward at the per-sample (re-spaced) timesteps, target = x_start.  The forward runs in the library, so
        the pair carries VALUES only (no autograd graph): it serves the loss terms of validation / evaluation
        (train_diffusion_smpl.py:66-120 computes them from this pair); optimising the weights is out of scope."""
        if self.loss_type not in (LossType.MSE, LossType.RESCALED_MSE):
            raise NotImplementedError(self.loss_type)
        if model_kwargs is None:
            model_kwargs = {}
        if noise is None:
            noise = th.randn_like(x_start)
        x_t = self.q_sample(x_start, t, noise=noise)
        y = model_kwargs["y"]
        if "inpainting_mask" in y.keys() and "inpainted_motion" in y.keys():
            m, gt = y["inpainting_mask"], y["inpainted_motion"]
            assert x_t.shape == m.shape == gt.shape
            x_t = (x_t * ~m) + (gt * m)
        ts = th.tensor(self.timestep_map, device=t.device, dtype=t.dtype)[t]       # _WrappedModel (respace.py:118-129)
        with th.no_grad():
            model_output = model(x_t, ts, **model_kwargs)
        target = x_start
        assert model_output.shape == target.shape == x_start.shape
        return model_output, target

    # ---- DDIM (gaussian_diffusion.py:738-999)
    def ddim_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None, eta=0.0, _noise=None):
        """ddim_sample (:738-788): model -> inpaint blend -> denoised_fn -> clamp, then eq. 12 through the engine's DDIM
        table (p_sample_finish).  With eta = 0 no noise is drawn (its coefficient is 0)."""
        if cond_fn is not None:
            raise NotImplementedError("cond_fn guidance is not on the reference's sampling path")
        eng, gt, mask = self._prepare(model, model_kwargs, T=x.shape[-1], kind=("ddim", float(eta)))
        i = self._uniform_step(t)
        x0 = eng.p_sample_predict(i, x, gt, mask)
        if denoised_fn is not None:
            x0 = denoised_fn(x0, t, model_kwargs)
        if clip_denoised:
            x0 = x0.clamp(-1, 1)
        noise = _noise
        if noise is None:
            noise = th.randn_like(x) if eta > 0 else th.zeros_like(x)
        return {"sample": eng.p_sample_finish(i, x0, x, noise), "pred_xstart": x0}

    def ddim_reverse_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None, eta=0.0):
        """ddim_reverse_sample (:847-883): x_t -> x_{t+1} along the deterministic ODE.  The model runs in the engine; the
        update is elementwise torch like q_sample."""
        assert eta == 0.0, "Reverse ODE only for deterministic path"
        eng, gt, mask = self._prepare(model, model_kwargs, T=x.shape[-1], kind=None)
        i = self._uniform_step(t)
        x0 = eng.p_sample_predict(i, x, gt, mask)
        if denoised_fn is not None:
            x0 = denoised_fn(x0, t, model_kwargs)
        if clip_denoised:
            x0 = x0.clamp(-1, 1)
        eps = ((_extract_into_tensor(self.sqrt_recip_alphas_cumprod, t, x.shape) * x - x0)
               / _extract_into_tensor(self.sqrt_recipm1_alphas_cumprod, t, x.shape))
        alpha_bar_next = _extract_into_tensor(self.alphas_cumprod_next, t, x.shape)
        mean_pred = x0 * th.sqrt(alpha_bar_next) + th.sqrt(1 - alpha_bar_next) * eps
        return {"sample": mean_pred, "pred_xstart": x0}

    def ddim_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                         device=None, progress=False, eta=0.0, skip_timesteps=0, init_image=None, randomize_class=False,
                         cond_fn_with_grad=False, dump_steps=None, const_noise=False):
        """ddim_sample_loop (:885-932).  Without a Python hook (or with the fused correction), progress bar, skipped steps or
        init image the whole loop runs in the library (idb_ddim_sample_loop, clip_denoised either way); otherwise step by
        step through ddim_sample_loop_progressive.  eta > 0 draws every step's noise up front in one generator call."""
        if dump_steps is not None:
            raise NotImplementedError()          # :909-910
        if const_noise:
            raise NotImplementedError()          # :911-912
        fused_hook = denoised_fn is None or getattr(denoised_fn, "is_fused_correction", False)
        if fused_hook and cond_fn is None and not progress and not skip_timesteps and init_image is None and not randomize_class \
                and not cond_fn_with_grad:
            eng, gt, mask = self._prepare(model, model_kwargs, T=shape[-1], kind=("ddim", float(eta)))
            x_T = noise if noise is not None else th.randn(*shape, device=eng.device)
            from ..sampling import draw_tape
            tape = draw_tape(eng, x_T, self.num_timesteps) if eta > 0 else None
            correction = denoised_fn is not None
            if correction:
                denoised_fn.bind(eng, model_kwargs)
            return eng.ddim_sample_loop(x_T, tape, gt, mask, correction=correction, clip_denoised=clip_denoised, use_graph=True)
        final = None
        for sample in self.ddim_sample_loop_progressive(
                model, shape, noise=noise, clip_denoised=clip_denoised, denoised_fn=denoised_fn, cond_fn=cond_fn,
                model_kwargs=model_kwargs, device=device, progress=progress, eta=eta, skip_timesteps=skip_timesteps,
                init_image=init_image, randomize_class=randomize_class, cond_fn_with_grad=cond_fn_with_grad):
            final = sample
        return final["sample"]

    def ddim_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                     model_kwargs=None, device=None, progress=False, eta=0.0, skip_timesteps=0, init_image=None,
                                     randomize_class=False, cond_fn_with_grad=False):
        """ddim_sample_loop_progressive (:934-999): unlike the DDPM loop there is no initial inpaint blend of x_T (:957-972;
        compare :694-699), and the steps are range(num_timesteps - skip_timesteps)[::-1] (:968)."""
        if cond_fn is not None or cond_fn_with_grad or randomize_class:
            raise NotImplementedError("classifier guidance options are not on the reference's sampling path")
        eng, gt, mask = self._prepare(model, model_kwargs, T=shape[-1], kind=("ddim", float(eta)))
        img = noise if noise is not None else th.randn(*shape, device=eng.device)
        if skip_timesteps and init_image is None:
            init_image = th.zeros_like(img)
        indices = list(range(self.num_timesteps - skip_timesteps))[::-1]
        if init_image is not None:
            img = self.q_sample(init_image, th.full((shape[0],), indices[0], device=eng.device, dtype=th.long), img)
        # eta > 0: every step's noise drawn up front in ONE generator call, exactly like the fused loop (same seed -> same
        # noise on both paths); the reference draws th.randn_like(x) per step (:779)
        from ..sampling import draw_tape
        tape = draw_tape(eng, img, len(indices)) if eta > 0 else None
        if progress:
            from tqdm.auto import tqdm
            indices = tqdm(indices)
        for k, i in enumerate(indices):
            t = th.full((shape[0],), i, device=eng.device, dtype=th.long)
            with th.no_grad():
                out = self.ddim_sample(model, img, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn, model_kwargs=model_kwargs,
                                       eta=eta, _noise=tape[k + 1] if tape is not None else None)
            yield out
            img = out["sample"]

    def _not_on_the_path(self, *a, **k):
        raise NotImplementedError("PLMS sampling is never called by the reference's scripts (SURVEY.md 2a #1)")

    plms_sample = plms_sample_loop = _not_on_the_path
