"""DDIM on the GPU through the C ABI (idb_diffusion_init_ddim, the per-step entries on a DDIM table, idb_ddim_sample_loop)
and through the mirrored SpacedDiffusion: teacher-forced steps and golden vectors against the reference's arithmetic,
bit-identity of the loop's execution paths, the correction hook, the free-running configs[1] chain, batch slices, the
graph cache across samplers, and the rejected arguments.  Tolerances: max|a-b| / max|b|."""
import json
import math
import os

import numpy as np
import pytest
import torch

from interdiff_b200 import synthetic as S
from interdiff_b200.engine import EngineError
from oracle import ddim as D
from oracle import restate as R
from tests.helpers import mdm_weights, projector_weights, rel
from tests.test_ddim import CASES, _key, _schedule, ddim_bound

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def eng():
    from interdiff_b200.engine import Engine
    e = Engine("cuda:0")
    yield e
    e.close()


def _setup(eng, B, T, source="auto"):
    sd = mdm_weights("smpl", source)
    eng.load_denoiser(sd, "smpl")
    b = S.make_smpl_batch(B=B, T=T)
    eng.bind(b["cond"], T)
    gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
    return sd, b, gt, mask


def _fwd(sd, cond):
    return lambda x, t: R.mdm_smpl_forward(sd, x, t, cond, faithful=False)


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_ddim_step_teacher_forced(eng, eta):
    """ddim50 of the 1000-step schedule: a spread of steps, each from the ORACLE's x_t, through idb_p_sample on the DDIM
    table; sample and pred_xstart within 2e-4 of ddim_sample_step"""
    sd, b, gt, mask = _setup(eng, 4, 30)
    betas, tmap = _schedule(1000, 50)
    eng.init_diffusion_ddim(betas, tmap, eta=eta)
    tb = D.ddim_tables(betas, eta, tmap)
    cond = torch.from_numpy(b["cond"])
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, len(betas)))
    x, worst = tape[0].clone(), 0.0
    for k, i in enumerate([49, 48, 40, 25, 10, 2, 1, 0]):
        noise = tape[k + 1]
        with torch.no_grad():
            ref, ref0 = D.ddim_sample_step(_fwd(sd, cond), tb, x, i, noise if eta > 0 else None, gt.cpu(), mask.cpu())
        got, got0 = eng.p_sample(i, x.cuda(), noise.cuda() if eta > 0 else torch.zeros_like(gt), gt, mask)
        worst = max(worst, rel(got, ref), rel(got0, ref0))
        x = ref
    assert worst < 2e-4, worst


@pytest.mark.parametrize("gemm", ["simt", "tcgen05"])
@pytest.mark.parametrize("source", ["random", "ref"])
def test_ddim_golden(gemm, source):
    """the whole loop against the reference's own ddim_sample_loop (ddim_smpl_*.npz), both GEMM backends"""
    from interdiff_b200.engine import Engine
    g = np.load(os.path.join(G, "ddim_smpl_%s.npz" % source))
    e = Engine("cuda:0")
    e.set_gemm_backend(gemm)
    _, b, gt, mask = _setup(e, 4, 30, source)
    betas, tmap = _schedule()
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, len(betas))).cuda()
    for eta, clip in CASES:
        e.init_diffusion_ddim(betas, tmap, eta=eta)
        got = e.ddim_sample_loop(tape[0], tape if eta > 0 else None, gt, mask, clip_denoised=clip).cpu()
        k = _key(eta, clip)
        assert rel(got, torch.from_numpy(g[k])) < ddim_bound(g, k), (k, rel(got, torch.from_numpy(g[k])))
    e.close()


def _mirror_steps(eng, x_T, tape, gt, mask, n, clip):
    """the step-by-step path of the mirror: predict -> clamp -> finish per step (noise zeros when there is no tape)"""
    x = x_T.clone()
    for k, i in enumerate(reversed(range(n))):
        x0 = eng.p_sample_predict(i, x, gt, mask)
        if clip:
            x0 = x0.clamp(-1, 1)
        x = eng.p_sample_finish(i, x0, x, tape[k + 1] if tape is not None else torch.zeros_like(x))
    return x


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_ddim_paths_bit_identical(eng, eta):
    """use_graph 0 / 1 / 2 and the step-by-step composition give the same bits, with clip on and off; eta = 0 without a
    tape equals eta = 0 fed a tape; the inpainted frames of the final sample are gt (clamped gt with clip)"""
    _, b, gt, mask = _setup(eng, 4, 30)
    betas, tmap = _schedule()
    n = len(betas)
    eng.init_diffusion_ddim(betas, tmap, eta=eta)
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, n)).cuda()
    x_T = tape[0].clone()
    finals = {}
    for clip in (False, True):
        outs = [eng.ddim_sample_loop(x_T, tape if eta > 0 else None, gt, mask, clip_denoised=clip, use_graph=m).clone()
                for m in (0, 1, 2)]
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), clip
        steps = _mirror_steps(eng, x_T, tape if eta > 0 else None, gt, mask, n, clip)
        assert torch.equal(outs[0], steps), clip
        if eta == 0:
            fed = eng.ddim_sample_loop(x_T, tape, gt, mask, clip_denoised=clip).clone()
            assert torch.equal(fed, outs[0]), clip
        want = gt.clamp(-1, 1) if clip else gt
        assert torch.equal(outs[0][mask], want[mask])
        finals[clip] = outs[0]
    if bool((gt[mask].abs() > 1).any()):
        assert not torch.equal(finals[False], finals[True])      # the clamp is observable on this batch


def test_ddim_loop_with_correction(eng, smplh_np):
    """52-step DDIM schedule, no respacing, eta = 0, tape-free: the fused hook runs at i = 50 and 0 with decisions exact
    against the oracle, and the fused loop equals the composition of the single-step entries bit for bit"""
    from tests.test_gpu_configs import _correction_ctx, _logging_denoised_fn
    B, T, steps = 3, 30, 52
    sd, b, gt, mask = _setup(eng, B, T, "random")
    psd = projector_weights("auto")
    eng.load_body(smplh_np)
    eng.load_projector(psd, 10, 20)
    eng.bind_correction(b["hand_pose"], b["betas"], b["obj_points"], past_len=10)
    betas = R.named_beta_schedule("cosine", steps)
    eng.init_diffusion_ddim(betas, eta=0.0)
    tb = D.ddim_tables(betas, 0.0)
    x_T = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    log = []
    with torch.no_grad():
        ref = D.ddim_sample_loop(_fwd(sd, torch.from_numpy(b["cond"])), tb, x_T, None, gt.cpu(), mask.cpu(),
                                 denoised_fn=_logging_denoised_fn(_correction_ctx(b, smplh_np, psd), log))
    assert [t for t, _, _ in log] == [50, 0]
    cond_log, contact_log = eng.correction_log(4)
    got = eng.ddim_sample_loop(x_T.cuda(), None, gt, mask, correction=True).clone()
    for k, (_, c_ref, ct_ref) in enumerate(log):
        assert torch.equal(cond_log[k].cpu().bool(), c_ref), k
        assert torch.equal(contact_log[k].cpu().long(), ct_ref), k
    assert int(cond_log[2:].sum()) == 0 and int(contact_log[2:].abs().sum()) == 0
    eng.correction_log(0)
    x = x_T.cuda()
    zeros = torch.zeros_like(x)
    for i in reversed(range(steps)):
        if i <= 500 and i % 50 == 0:
            x0 = eng.p_sample_predict(i, x, gt, mask)
            eng.correction_apply(x0, gt, i)
            x = eng.p_sample_finish(i, x0, x, zeros)
        else:
            x, _ = eng.p_sample(i, x, zeros, gt, mask)
    assert torch.equal(got, x)
    assert rel(got, ref) < 1e-3


def test_ddim50_free_running_configs1(eng, record_property):
    """configs[1] (B=64, T=30, shipped checkpoint where exported), ddim50 of the 100-step schedule at eta = 0, free-running
    against the oracle: <= 1e-3 per step up to the step where the reference's own float32 and float64 runs disagree by more
    than 1e-4 (tests/golden/ddim_conditioning.json, a CPU run of oracle/ddim_conditioning_probe.py); the rest is recorded
    as a curve (test property `ddim50_curve`, e.g. in the --junitxml report).  The fused loop is the same computation as the chain of single steps."""
    B, T = 64, 30
    sd, b, gt, mask = _setup(eng, B, T, "auto")
    betas, tmap = _schedule(100, 50)
    eng.init_diffusion_ddim(betas, tmap, eta=0.0)
    tb = D.ddim_tables(betas, 0.0, tmap)
    x_T = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    torch.set_num_threads(min(os.cpu_count(), 32))
    with torch.no_grad():
        _, traj = D.ddim_sample_loop(_fwd(sd, torch.from_numpy(b["cond"])), tb, x_T, None, gt.cpu(), mask.cpu(), return_trajectory=True)
    x, zeros, curve = x_T.cuda(), torch.zeros_like(gt), []
    for k, i in enumerate(reversed(range(len(betas)))):
        x, _ = eng.p_sample(i, x, zeros, gt, mask)
        curve.append(rel(x, traj[k][0]))
    with open(os.path.join(G, "ddim_conditioning.json")) as f:
        probe = json.load(f)["spacings"]["ddim50"]
    cut = int(probe["first_step_above_1e4"])
    record_property("ddim50_curve", json.dumps(dict(free_running_vs_oracle=curve, reference_f32_vs_f64=probe["reference_f32_vs_f64"],
                                                    cutoff_step=cut)))
    bad = [(k, v) for k, v in enumerate(curve[:cut]) if v > 1e-3]
    assert not bad, (bad[:5], cut)
    fused = eng.ddim_sample_loop(x_T.cuda(), None, gt, mask)
    assert rel(fused, x) < 1e-6
    assert torch.equal(fused[mask], gt[mask])


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_ddim_batch_slices_bit_identical(eng, eta):
    """slices of one global B=64 batch reproduce the full batch bit for bit (eta 0.5: noise keyed by the global sample
    index through draw_tape_indexed)"""
    from interdiff_b200.sampling import draw_tape_indexed
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    B, T = 64, 30
    b = S.make_smpl_batch(B=B, T=T)
    betas, tmap = _schedule()
    eng.init_diffusion_ddim(betas, tmap, eta=eta)
    gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
    tape = draw_tape_indexed(eng, (1, 144, T), len(betas), list(range(B)), seed=233)
    use = tape if eta > 0 else None
    eng.bind(b["cond"], T)
    full = eng.ddim_sample_loop(tape[0], use, gt, mask).clone()
    for G_ in (2, 8):
        n = B // G_
        parts = []
        for r in range(G_):
            sl = slice(r * n, (r + 1) * n)
            eng.bind(np.ascontiguousarray(b["cond"][:, sl]), T)
            t_r = draw_tape_indexed(eng, (1, 144, T), len(betas), list(range(sl.start, sl.stop)), seed=233)
            assert torch.equal(t_r, tape[:, sl])
            parts.append(eng.ddim_sample_loop(t_r[0], t_r if eta > 0 else None, gt[sl].contiguous(), mask[sl].contiguous()).clone())
        assert torch.equal(torch.cat(parts, dim=0), full), G_


def test_graph_cache_across_samplers(eng):
    """one engine alternating DDPM <-> DDIM, eta and clip, with the whole-loop and per-step graphs, gives what a fresh
    engine gives for each configuration (no stale graph is replayed)"""
    from interdiff_b200.engine import Engine
    sd, b, gt, mask = _setup(eng, 4, 30)
    betas, tmap = _schedule()
    n = len(betas)
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, n)).cuda()
    runs = [("ddim", 0.0, False), ("ddpm", None, False), ("ddim", 0.0, True), ("ddim", 0.5, True), ("ddim", 0.5, False),
            ("ddpm", None, False), ("ddim", 0.0, False)]

    def run(e, kind, eta, clip, mode):
        if kind == "ddpm":
            e.init_diffusion(betas, tmap)
            return e.p_sample_loop(tape, gt, mask, use_graph=mode).clone()
        e.init_diffusion_ddim(betas, tmap, eta=eta)
        return e.ddim_sample_loop(tape[0], tape if eta > 0 else None, gt, mask, clip_denoised=clip, use_graph=mode).clone()
    fresh = {}
    for cfg in set(runs):
        e = Engine("cuda:0")
        e.load_denoiser(sd, "smpl")
        e.bind(b["cond"], 30)
        fresh[cfg] = run(e, *cfg, "off")
        e.close()
    for mode in ("loop", "step"):
        for cfg in runs:
            assert torch.equal(run(eng, *cfg, mode), fresh[cfg]), (mode, cfg)
    # clip toggled without re-initialising the table: the graphs are keyed on it
    eng.init_diffusion_ddim(betas, tmap, eta=0.0)
    for mode in ("loop", "step"):
        for clip in (True, False, True):
            assert torch.equal(eng.ddim_sample_loop(tape[0], None, gt, mask, clip_denoised=clip, use_graph=mode), fresh[("ddim", 0.0, clip)])
    assert not torch.equal(fresh[("ddim", 0.0, False)], fresh[("ddpm", None, False)])


def _status(excinfo):
    return int(str(excinfo.value).rsplit("status ", 1)[1].rstrip(")"))


def test_ddim_errors_leave_the_engine_usable(eng):
    _, b, gt, mask = _setup(eng, 4, 30)
    betas, tmap = _schedule()
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, len(betas))).cuda()
    eng.init_diffusion_ddim(betas, tmap, eta=0.0)
    want = eng.ddim_sample_loop(tape[0], None, gt, mask).clone()
    for bad in (-0.5, float("nan"), float("inf"), 5.0):          # eta = 5: 1 - alpha_bar_prev - sigma^2 < 0
        with pytest.raises(EngineError) as ei:
            eng.init_diffusion_ddim(betas, tmap, eta=bad)
        assert _status(ei) == 2, bad
        assert torch.equal(eng.ddim_sample_loop(tape[0], None, gt, mask), want), bad      # the loaded table is kept
    eng.init_diffusion_ddim(betas, tmap, eta=0.5)
    with pytest.raises(EngineError) as ei:
        eng.ddim_sample_loop(tape[0], None, gt, mask)                # sigma != 0 needs a tape
    assert _status(ei) == 2
    noisy = eng.ddim_sample_loop(tape[0], tape, gt, mask).clone()
    assert torch.isfinite(noisy).all() and not torch.equal(noisy, want)
    eng.init_diffusion(betas, tmap)
    with pytest.raises(EngineError) as ei:
        eng.ddim_sample_loop(tape[0], tape, gt, mask)               # a DDPM table is loaded
    assert _status(ei) == 3
    ddpm = eng.p_sample_loop(tape, gt, mask).clone()
    assert torch.isfinite(ddpm).all()
    eng.init_diffusion_ddim(betas, tmap, eta=0.0)
    assert torch.equal(eng.ddim_sample_loop(tape[0], None, gt, mask), want)


def test_mirror_ddim_end_to_end():
    """SpacedDiffusion(space_timesteps(100, "ddim10")) of the mirror on the mirrored MDM: ddim_sample_loop fused (no hook) and
    step by step (plain-Python denoised_fn), clip on and off, eta 0 and 0.5, against the oracle; ddim_reverse_sample against
    the oracle's reverse step"""
    from interdiff_b200.diffusion import gaussian_diffusion as gd
    from interdiff_b200.diffusion.respace import SpacedDiffusion, space_timesteps
    from tests.test_gpu_configs import _mirror_model
    model, _, msd = _mirror_model(100, "random")
    diffusion = SpacedDiffusion(space_timesteps(100, "ddim10"), betas=gd.get_named_beta_schedule("cosine", 100),
                                model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    b = S.make_smpl_batch(B=3, T=30)
    cond, gt, mask = (torch.from_numpy(b[k]).cuda() for k in ("cond", "gt", "mask"))
    kw = {"y": {"cond": cond, "inpainted_motion": gt, "inpainting_mask": mask}}
    x_T = torch.randn(gt.shape, generator=torch.Generator().manual_seed(3)).cuda()
    cpu_sd = {k: v.cpu() for k, v in msd.items()}
    fwd = _fwd(cpu_sd, cond.cpu())
    identity = lambda x, t, model_kwargs: x
    for eta in (0.0, 0.5):
        for clip in (False, True):
            torch.manual_seed(11)
            fused = diffusion.ddim_sample_loop(model, gt.shape, noise=x_T, clip_denoised=clip, model_kwargs=kw, eta=eta).clone()
            torch.manual_seed(11)
            stepped = diffusion.ddim_sample_loop(model, gt.shape, noise=x_T, clip_denoised=clip, model_kwargs=kw, eta=eta,
                                                 denoised_fn=identity).clone()
            assert torch.equal(fused, stepped), (eta, clip)
            tape = None
            if eta > 0:          # the tape both paths drew: same seed, same single generator call
                from interdiff_b200.sampling import draw_tape
                torch.manual_seed(11)
                tape = draw_tape(model.engine_for(cond.device), x_T, 10).cpu()
            tb = D.ddim_tables(diffusion.betas, eta, diffusion.timestep_map)
            with torch.no_grad():
                ref = D.ddim_sample_loop(fwd, tb, x_T.cpu(), tape, gt.cpu(), mask.cpu(), clip_denoised=clip)
            assert rel(fused, ref) < 1e-3, (eta, clip, rel(fused, ref))
    # the default clip_denoised is True, as in the reference (:890)
    torch.manual_seed(11)
    assert torch.equal(diffusion.ddim_sample_loop(model, gt.shape, noise=x_T, model_kwargs=kw),
                       diffusion.ddim_sample_loop(model, gt.shape, noise=x_T, model_kwargs=kw, clip_denoised=True))
    # ddim_reverse_sample: one step x_t -> x_{t+1} from a noised gt, i = 4 and 0
    tb = D.ddim_tables(diffusion.betas, 0.0, diffusion.timestep_map)
    for i in (4, 0):
        a = math.sqrt(tb["alphas_cumprod"][i])
        x = a * gt + math.sqrt(1 - a * a) * torch.randn(gt.shape, generator=torch.Generator().manual_seed(i)).cuda()
        out = diffusion.ddim_reverse_sample(model, x, torch.full((3,), i, device="cuda"), clip_denoised=False, model_kwargs=kw)
        with torch.no_grad():
            ref, ref0 = D.ddim_reverse_step(fwd, tb, x.cpu(), i, gt.cpu(), mask.cpu())
        assert rel(out["pred_xstart"], ref0) < 2e-4 and rel(out["sample"], ref) < 2e-4, i
