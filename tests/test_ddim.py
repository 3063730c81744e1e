"""DDIM on the CPU: the oracle's tables, step and loop (oracle/restate.py) against the reference's own ddim_sample
(golden vectors written by `python -m oracle.make_golden_ddim`, and the live tree where it is installed), and the
mirror's argument handling where the reference raises.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from interdiff_b200 import synthetic as S
from oracle import ddim as D
from oracle import restate as R
from tests.helpers import mdm_weights, rel

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = [(eta, clip) for eta in (0.0, 0.5) for clip in (False, True)]


def _key(eta, clip):
    return "eta%g_clip%d" % (eta, int(clip))


def _schedule(n=100, count=10):
    return D.respace(R.named_beta_schedule("cosine", n), D.ddim_use_timesteps(n, count))


@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_ddim_tables_match_the_reference_formulas(eta):
    """the folded (a, b, sigma_nz) reproduce ddim_sample's eq. 12 (gaussian_diffusion.py:769-787) evaluated directly in
    float64 on random (x0, x_t, noise); at i = 0 the update is x0 exactly"""
    betas, tmap = _schedule(1000, 50)
    tb = D.ddim_tables(betas, eta, tmap)
    assert tb["timestep_map"] == sorted(D.ddim_use_timesteps(1000, 50))
    ac = np.cumprod(1.0 - betas)
    ac_prev = np.append(1.0, ac[:-1])
    g = np.random.default_rng(0)
    x0, xt, nz = g.standard_normal((3, len(betas), 64))
    for i in range(len(betas)):
        eps = (np.sqrt(1.0 / ac[i]) * xt[i] - x0[i]) / np.sqrt(1.0 / ac[i] - 1)
        sigma = eta * np.sqrt((1 - ac_prev[i]) / (1 - ac[i])) * np.sqrt(1 - ac[i] / ac_prev[i])
        want = x0[i] * np.sqrt(ac_prev[i]) + np.sqrt(1 - ac_prev[i] - sigma ** 2) * eps + (i != 0) * sigma * nz[i]
        got = tb["a"][i] * x0[i] + tb["b"][i] * xt[i] + tb["sigma_nz"][i] * nz[i]
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), i
    assert tb["a"][0] == 1.0 and tb["b"][0] == 0.0 and tb["sigma_nz"][0] == 0.0 and tb["sigma"][0] == 0.0
    if eta == 0.0:
        assert not tb["sigma_nz"].any()


def _oracle_loop(sd, b, eta, clip, dtype=torch.float32):
    betas, tmap = _schedule()
    tb = D.ddim_tables(betas, eta, tmap)
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, 10)).to(dtype)
    cond, gt, mask = torch.from_numpy(b["cond"]).to(dtype), torch.from_numpy(b["gt"]).to(dtype), torch.from_numpy(b["mask"])
    if dtype == torch.float64:
        sd = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad():
        return D.ddim_sample_loop(lambda x, t: R.mdm_smpl_forward(sd, x, t, cond, faithful=False), tb, tape[0],
                                  tape if eta > 0 else None, gt, mask, clip_denoised=clip)


def ddim_bound(g, key):
    """parity bound against the reference's float32 loop: 3e-3 (test_golden.py's bound for short loops), widened where the
    golden file also stores the reference's float64 runs (shipped checkpoint) to 3x the largest distance between the
    reference's own float32 and float64 runs over the four cases: that spread (6e-4 .. 3e-2 for the ddim10 chain) measures
    how far the chain carries float32 rounding, and where a float32 implementation lands inside it is a matter of luck"""
    spreads = [rel(torch.from_numpy(g[k]), torch.from_numpy(g[k + "_f64"])) for k in (_key(e, c) for e, c in CASES) if k + "_f64" in g]
    return max([3e-3] + [3.0 * v for v in spreads])


@pytest.mark.parametrize("source", ["random", "ref"])
def test_oracle_ddim_loop_matches_golden(source):
    """the oracle loop against the reference's own SpacedDiffusion.ddim_sample_loop ("ddim10" of a 100-step cosine schedule,
    B=4, T=30, inpainting), eta in {0, 0.5} x clip_denoised in {False, True}"""
    g = np.load(os.path.join(G, "ddim_smpl_%s.npz" % source))
    sd = mdm_weights("smpl", source)
    b = S.make_smpl_batch(B=4, T=30)
    assert list(g["timestep_map"]) == _schedule()[1]
    for eta, clip in CASES:
        k = _key(eta, clip)
        out = _oracle_loop(sd, b, eta, clip)
        # seeded weights: measured 2.2e-6; shipped checkpoint: within the reference's own float32 / float64 spread
        bound = 1e-5 if source == "random" else ddim_bound(g, k)
        assert rel(out, torch.from_numpy(g[k])) < bound, (k, rel(out, torch.from_numpy(g[k])), bound)
        if k + "_f64" in g:
            # float64 oracle vs the reference's float64 run (which extracts its coefficients as float32, :1611-1623)
            out64 = _oracle_loop(sd, b, eta, clip, torch.float64)
            assert rel(out64, torch.from_numpy(g[k + "_f64"])) < 3e-3, k
        gt = torch.from_numpy(b["gt"])
        want = gt.clamp(-1, 1) if clip else gt          # i = 0: a = 1, b = 0 -> the inpainted frames are pred_xstart's
        assert torch.equal(out[b["mask"]], want[b["mask"]])


def _reference():
    from oracle import ref_loader as RL
    if not RL.available():
        pytest.skip("reference tree not installed")
    return RL


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_oracle_ddim_step_matches_live_reference(eta, clip):
    """one ddim_sample of the reference (model wrapped by SpacedDiffusion) against ddim_sample_step, same x_t and noise"""
    RL = _reference()
    from oracle import make_golden_ddim as MG
    sd = mdm_weights("smpl", "random")
    model, _, _ = RL.build_mdm_smpl(state_dict=sd, diffusion_steps=100)
    diffusion = MG.reference_ddim_diffusion(100, "ddim10")
    gd = RL.modules()["diffusion.gaussian_diffusion"]
    b = S.make_smpl_batch(B=3, T=30)
    cond, gt, mask = torch.from_numpy(b["cond"]), torch.from_numpy(b["gt"]), torch.from_numpy(b["mask"])
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, 2))
    betas, tmap = _schedule()
    assert list(diffusion.timestep_map) == tmap
    tb = D.ddim_tables(betas, eta, tmap)
    kw = {"y": {"cond": cond, "inpainted_motion": gt, "inpainting_mask": mask}}
    for i in (9, 4, 0):
        old, gd.th.randn_like = gd.th.randn_like, (lambda x_: tape[1].clone())
        try:
            with torch.no_grad():
                ref = diffusion.ddim_sample(model, tape[0], torch.full((3,), i), clip_denoised=clip, model_kwargs=kw, eta=eta)
        finally:
            gd.th.randn_like = old
        with torch.no_grad():
            got, got0 = D.ddim_sample_step(lambda x, t: R.mdm_smpl_forward(sd, x, t, cond), tb, tape[0], i, tape[1], gt, mask,
                                           clip_denoised=clip)
        assert rel(got0, ref["pred_xstart"]) < 1e-5 and rel(got, ref["sample"]) < 1e-5, i


def _mirror_diffusion(steps=100, spacing="ddim10"):
    from interdiff_b200.diffusion import gaussian_diffusion as gd
    from interdiff_b200.diffusion.respace import SpacedDiffusion, space_timesteps
    return SpacedDiffusion(space_timesteps(steps, spacing), betas=gd.get_named_beta_schedule("cosine", steps),
                           model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)


def test_mirror_respacing_and_tables_match_the_oracle():
    d = _mirror_diffusion()
    betas, tmap = _schedule()
    assert d.timestep_map == tmap and np.array_equal(d.betas, betas)
    tb = D.ddim_tables(betas, 0.0, tmap)
    for name in ("alphas_cumprod_next", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod"):
        assert np.array_equal(getattr(d, name), tb[name]), name


def test_mirror_raises_where_the_reference_raises():
    """ddim_sample_loop: dump_steps and const_noise=True raise NotImplementedError before anything runs (:909-912); PLMS is
    not built; ddim_reverse_sample asserts eta == 0 (:860)"""
    d = _mirror_diffusion()
    shape = (2, 1, 144, 30)
    with pytest.raises(NotImplementedError):
        d.ddim_sample_loop(object(), shape, dump_steps=[1])
    with pytest.raises(NotImplementedError):
        d.ddim_sample_loop(object(), shape, const_noise=True)
    for fn in (d.plms_sample, d.plms_sample_loop):
        with pytest.raises(NotImplementedError):
            fn(object(), shape)
    with pytest.raises(AssertionError):
        d.ddim_reverse_sample(object(), torch.zeros(shape), torch.zeros(2, dtype=torch.long), eta=0.5)
    # models that are not interdiff_b200 models are refused (no eager fallback)
    with pytest.raises(TypeError):
        d.ddim_sample_loop(object(), shape, model_kwargs={"y": {}})
