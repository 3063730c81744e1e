"""CPU restatement (torch) of the reference's DDIM sampler for the START_X model: ddim_sample, ddim_reverse_sample and
ddim_sample_loop(_progressive) (diffusion/gaussian_diffusion.py:738-999) on a schedule re-spaced as SpacedDiffusion does
(diffusion/respace.py:8-87).  TEST INFRASTRUCTURE like oracle/restate.py (which provides the denoiser and the beta
schedules): the parity checker of the CUDA DDIM path; the product never imports it.

Pinned by tests/test_ddim.py against the golden vectors of oracle/make_golden_ddim.py (the reference's own classes) and
against the live reference where the tree is installed.
"""
import numpy as np
import torch


def ddim_use_timesteps(n, count):
    """space_timesteps(n, "ddim<count>") (respace.py:31-38): the integer stride that gives exactly `count` steps."""
    for stride in range(1, n):
        if len(range(0, n, stride)) == count:
            return set(range(0, n, stride))
    raise ValueError("cannot create exactly %d steps with an integer stride" % count)


def respace(betas, use_timesteps):
    """SpacedDiffusion.__init__ (respace.py:73-87): (re-spaced float64 betas, timestep_map)."""
    ac = np.cumprod(1.0 - np.asarray(betas, dtype=np.float64))
    last, new_betas, tmap = 1.0, [], []
    for i, a in enumerate(ac):
        if i in use_timesteps:
            new_betas.append(1 - a / last)
            last = a
            tmap.append(i)
    return np.array(new_betas), tmap


def ddim_tables(betas, eta, timestep_map=None):
    """Float64 tables of ddim_sample (gaussian_diffusion.py:769-787) for the (re-spaced) betas: the reference's own
    arrays (alphas_cumprod, alphas_cumprod_prev, sqrt_recip(m1)_alphas_cumprod, :160-197) plus sigma and the update
    folded onto (x0, x_t): x_prev = a x0 + b x_t + sigma_nz noise, with k = sqrt(1 - ac_prev - sigma^2),
    a = sqrt(ac_prev) - k / sqrt_recipm1, b = k sqrt_recip / sqrt_recipm1, sigma_nz = 1[i != 0] sigma."""
    betas = np.asarray(betas, dtype=np.float64)
    ac = np.cumprod(1.0 - betas)
    ac_prev = np.append(1.0, ac[:-1])
    sqrt_recip, sqrt_recipm1 = np.sqrt(1.0 / ac), np.sqrt(1.0 / ac - 1)
    sigma = eta * np.sqrt((1 - ac_prev) / (1 - ac)) * np.sqrt(1 - ac / ac_prev)
    k = np.sqrt(1 - ac_prev - sigma ** 2)
    n = len(betas)
    return dict(betas=betas, eta=float(eta), timestep_map=list(timestep_map) if timestep_map is not None else list(range(n)),
                alphas_cumprod=ac, alphas_cumprod_prev=ac_prev, alphas_cumprod_next=np.append(ac[1:], 0.0),
                sqrt_recip_alphas_cumprod=sqrt_recip, sqrt_recipm1_alphas_cumprod=sqrt_recipm1, sigma=sigma,
                a=np.sqrt(ac_prev) - k / sqrt_recipm1, b=k * sqrt_recip / sqrt_recipm1, sigma_nz=np.where(np.arange(n) == 0, 0.0, sigma))


def _extract(arr, i, dtype):
    """_extract_into_tensor (:1611-1623) of one uniform step: float64 -> .float(); a float64 run keeps float64 (the
    rounding-free yardstick)"""
    return torch.tensor(float(arr[i]), dtype=torch.float64 if dtype == torch.float64 else torch.float32)


def ddim_sample_step(model_fn, tables, x, i, noise=None, gt=None, mask=None, denoised_fn=None, model_kwargs=None,
                     clip_denoised=False):
    """One ddim_sample (gaussian_diffusion.py:738-788) for a uniform step index i, in the reference's arithmetic order:
    model(x, timestep_map[i]) -> inpaint blend (:307-311) -> denoised_fn (with the UN-mapped i, :356) -> clamp ->
    eps re-derived from x0 (:407-411) -> sigma, eq. 12, + 1[i != 0] sigma noise.  noise may be None when eta = 0.
    Dtype-generic: float32 inputs reproduce the reference, float64 inputs give the yardstick.  Returns (sample, pred_xstart)."""
    B, dt = x.shape[0], x.dtype
    t = torch.full((B,), int(i), dtype=torch.long)
    out = model_fn(x, torch.full((B,), int(tables["timestep_map"][i]), dtype=torch.long))
    if mask is not None and gt is not None:
        out = (out * ~mask) + (gt * mask)
    if denoised_fn is not None:
        out = denoised_fn(out, t, model_kwargs)
    if clip_denoised:
        out = out.clamp(-1, 1)
    eps = (_extract(tables["sqrt_recip_alphas_cumprod"], i, dt) * x - out) / _extract(tables["sqrt_recipm1_alphas_cumprod"], i, dt)
    alpha_bar, alpha_bar_prev = _extract(tables["alphas_cumprod"], i, dt), _extract(tables["alphas_cumprod_prev"], i, dt)
    sigma = tables["eta"] * torch.sqrt((1 - alpha_bar_prev) / (1 - alpha_bar)) * torch.sqrt(1 - alpha_bar / alpha_bar_prev)
    sample = out * torch.sqrt(alpha_bar_prev) + torch.sqrt(1 - alpha_bar_prev - sigma ** 2) * eps
    if noise is not None:
        sample = sample + (0.0 if i == 0 else 1.0) * sigma * noise
    return sample, out


def ddim_reverse_step(model_fn, tables, x, i, gt=None, mask=None, clip_denoised=False):
    """ddim_reverse_sample (gaussian_diffusion.py:847-883), eta = 0: x_t -> x_{t+1}.  Returns (sample, pred_xstart)."""
    dt = x.dtype
    out = model_fn(x, torch.full((x.shape[0],), int(tables["timestep_map"][i]), dtype=torch.long))
    if mask is not None and gt is not None:
        out = (out * ~mask) + (gt * mask)
    if clip_denoised:
        out = out.clamp(-1, 1)
    eps = (_extract(tables["sqrt_recip_alphas_cumprod"], i, dt) * x - out) / _extract(tables["sqrt_recipm1_alphas_cumprod"], i, dt)
    alpha_bar_next = _extract(tables["alphas_cumprod_next"], i, dt)
    return out * torch.sqrt(alpha_bar_next) + torch.sqrt(1 - alpha_bar_next) * eps, out


def ddim_sample_loop(model_fn, tables, x_T, tape=None, gt=None, mask=None, denoised_fn=None, model_kwargs=None, clip_denoised=False,
                     return_trajectory=False):
    """ddim_sample_loop(_progressive) (gaussian_diffusion.py:885-999) with caller-provided x_T: no initial inpaint blend
    (:957-972), steps i = n-1 .. 0; tape[k + 1] = noise of the k-th step (None: eta = 0, no noise term)."""
    n = len(tables["betas"])
    x = x_T.clone()
    traj = []
    for k, i in enumerate(reversed(range(n))):
        x, x0 = ddim_sample_step(model_fn, tables, x, i, tape[k + 1] if tape is not None else None, gt, mask, denoised_fn,
                                 model_kwargs, clip_denoised)
        if return_trajectory:
            traj.append((x.clone(), x0.clone()))
    return (x, traj) if return_trajectory else x
