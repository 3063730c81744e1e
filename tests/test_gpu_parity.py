"""GPU parity: the CUDA path (through the C ABI) against oracle.restate on the same seeded
inputs.  Tolerances are max-norm relative, max|a-b| / max|b| (SURVEY 8d "Parity check"); the
north-star bound is 1e-3, the bounds asserted here are the tighter ones an fp32-grade
implementation should meet."""
import numpy as np
import pytest
import torch

from interdiff_b200 import synthetic as S
from oracle import restate as R
from tests.helpers import encoder_weights, mdm_weights, projector_weights, rel, smplh_torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["simt", "tcgen05"])
def eng(request):
    """Every parity test runs with both GEMM backends (fp32 SIMT and tcgen05 split-precision; the latter includes the fused feed-forward cluster kernel)."""
    from interdiff_b200.engine import Engine
    e = Engine("cuda:0")
    e.set_gemm_backend(request.param)
    yield e
    e.close()


@pytest.mark.parametrize("source", ["random", "ref"])
@pytest.mark.parametrize("rotary", ["absolute", "bucketed"])
def test_denoiser_forward_smpl(eng, source, rotary):
    sd = mdm_weights("smpl", source)
    eng.load_denoiser(sd, "smpl", rotary=rotary)
    B, T = 5, 30
    b = S.make_smpl_batch(B=B, T=T)
    eng.bind(b["cond"], T)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([999, 500, 37, 1, 0])
    got = eng.forward(x.cuda(), t.cuda()).cpu()
    with torch.no_grad():
        ref = R.mdm_smpl_forward(sd, x, t, torch.from_numpy(b["cond"]), rotary=rotary, faithful=True)
    assert rel(got, ref) < 2e-4


@pytest.mark.parametrize("B,Tp", [(5, 10), (3, 16)])
def test_condition_encoder(eng, B, Tp):
    """conditioning encoder (past frames + point-cloud embedding -> cond) against the oracle, then straight into
    bind + forward: the memory produced on the device drives the decoder exactly like a host-provided one"""
    sd = encoder_weights("auto")
    eng.load_denoiser(sd, "smpl")
    b = S.make_smpl_batch(B=B, T=30)
    past = torch.from_numpy(b["gt"])[..., :Tp].contiguous()
    pc = torch.randn(B, 256, generator=torch.Generator().manual_seed(B))
    cond = eng.encode_condition(past.cuda(), pc.cuda())
    with torch.no_grad():
        ref = R.mdm_smpl_condition(sd, past, pc, faithful=False)
    assert rel(cond.cpu(), ref) < 2e-4
    eng.bind(cond, 30)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.full((B,), 321)
    got = eng.forward(x.cuda(), t.cuda()).cpu()
    with torch.no_grad():
        want = R.mdm_smpl_forward(sd, x, t, ref, faithful=False)
    assert rel(got, want) < 3e-4


@pytest.mark.parametrize("P", [2048, 1000])
def test_pointcloud_encoder(eng, P):
    """PointNet++ point-cloud encoder against the oracle on clouds that exercise the operator corner cases: points
    inside the |p|^2 <= 1e-3 dead zone of the sampler, duplicated points (distance ties), a cloud size that is not a
    multiple of the sampler's block."""
    from oracle import pointnet2_restated as P2
    sd = encoder_weights("auto")
    eng.load_denoiser(sd, "smpl")
    g = torch.Generator().manual_seed(P)
    B = 3
    pts = 0.25 * (torch.rand(B, P, 3, generator=g) - 0.5) * torch.tensor([1.0, 2.0, 0.7])
    pts[:, 5] = 0.01 * torch.randn(B, 3, generator=g)        # inside the dead zone
    pts[:, 77] = pts[:, 76]                                    # duplicates
    pts[1, 300:310] = pts[1, 100:110]
    got = eng.pointcloud_embed(pts.cuda()).cpu()
    with torch.no_grad():
        ref = P2.pointnet2_encoder(sd, pts)
    assert rel(got, ref) < 1e-4


def test_mirror_get_embeddings():
    """interdiff_b200.model.diffusion_smpl.MDM._get_embeddings (reference API: list of per-frame dicts) with the
    point-cloud embedding supplied: axis-angle -> rot6d plumbing on the host side + the encoder in the library,
    against oracle.transforms + oracle.restate on the same weights."""
    from argparse import Namespace
    from interdiff_b200.model.diffusion_smpl import MDM
    from oracle import transforms as tf
    from tests.test_host_api import SMPL_ARGS
    sd = encoder_weights("auto")
    m = MDM(Namespace(**{**SMPL_ARGS, "future_len": 20})).cuda().eval()
    own = m.state_dict()
    m.load_state_dict({k: (sd[k].reshape(own[k].shape) if k in sd else v) for k, v in own.items()})
    g = torch.Generator().manual_seed(9)
    T, B = 30, 3
    frames = [dict(smplfit_params=dict(pose=0.4 * torch.randn(B, 156, generator=g), trans=torch.randn(B, 3, generator=g)),
                   objfit_params=dict(angle=0.7 * torch.randn(B, 3, generator=g), trans=torch.randn(B, 3, generator=g))) for _ in range(T)]
    pc = torch.randn(B, 256, generator=g)
    cond, gt = m._get_embeddings(dict(frames=frames, pc_embedding=pc), device="cuda")
    # ... and with the point cloud itself: PointNet++ runs in the library as well
    from oracle import pointnet2_restated as P2
    pts = 0.2 * (torch.rand(B, 2048, 3, generator=g) - 0.5)
    cond_pts, _ = m._get_embeddings(dict(frames=frames, obj_points=torch.cat([pts, torch.zeros(B, 2048, 4)], dim=2)), device="cuda")
    pose = torch.stack([f["smplfit_params"]["pose"][:, :66] for f in frames])
    r6 = lambda aa: tf.matrix_to_rotation_6d(tf.axis_angle_to_matrix(aa))
    gt_ref = torch.cat([r6(pose.view(T, B, 22, 3)).reshape(T, B, 132), torch.stack([f["smplfit_params"]["trans"] for f in frames]),
                        r6(torch.stack([f["objfit_params"]["angle"] for f in frames]).view(T, B, 1, 3)).reshape(T, B, 6),
                        torch.stack([f["objfit_params"]["trans"] for f in frames])], dim=2)
    assert rel(gt.cpu(), gt_ref) < 1e-5
    past = gt_ref[:10].permute(1, 2, 0).unsqueeze(1).contiguous()
    with torch.no_grad():
        msd = {k: v.cpu() for k, v in m.state_dict().items()}
        ref = R.mdm_smpl_condition(msd, past, pc, faithful=False)
        ref_pts = R.mdm_smpl_condition(msd, past, P2.pointnet2_encoder(msd, pts), faithful=False)
    assert rel(cond.cpu(), ref) < 2e-4
    assert rel(cond_pts.cpu(), ref_pts) < 2e-4


def test_denoiser_forward_T35(eng):
    """default reference window (past 10 + future 25), T > 32 exercises the strided loops"""
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    B, T = 3, 35
    b = S.make_smpl_batch(B=B, T=T)
    eng.bind(b["cond"], T)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([800, 20, 3])
    got = eng.forward(x.cuda(), t.cuda()).cpu()
    with torch.no_grad():
        ref = R.mdm_smpl_forward(sd, x, t, torch.from_numpy(b["cond"]), faithful=False)
    assert rel(got, ref) < 2e-4


@pytest.mark.parametrize("T,Tm", [(36, 16), (17, 3), (16, 9)])
def test_denoiser_forward_window_extremes(eng, T, Tm):
    """largest supported window / memory (maximum shared-memory footprint of the attention kernels, two
    key tiles per warp group), a short odd one, and an exact single slab"""
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    B = 3
    b = S.make_smpl_batch(B=B, T=T)
    cond = np.random.default_rng(T * 100 + Tm).standard_normal((Tm, B, 256)).astype(np.float32)
    eng.bind(cond, T)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([640, 77, 0])
    got = eng.forward(x.cuda(), t.cuda()).cpu()
    with torch.no_grad():
        ref = R.mdm_smpl_forward(sd, x, t, torch.from_numpy(cond), faithful=False)
    assert rel(got, ref) < 2e-4


@pytest.mark.parametrize("source", ["random", "ref"])
def test_denoiser_forward_skeleton(eng, source):
    """BASELINE config 1: skeleton diffusion, B=2, T=15."""
    sd = mdm_weights("skeleton", source)
    eng.load_denoiser(sd, "skeleton")
    b = S.make_skeleton_batch(B=2, T=15)
    eng.bind(b["cond"], 15, zero_pose_obj=b["zero_pose_obj"])
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([999, 4])
    got = eng.forward(x.cuda(), t.cuda()).cpu()
    with torch.no_grad():
        ref = R.mdm_skeleton_forward(sd, x, t, torch.from_numpy(b["zero_pose_obj"]), torch.from_numpy(b["cond"]))
    assert rel(got, ref) < 2e-4


def _loop_setup(eng, B, T, steps, source="auto"):
    sd = mdm_weights("smpl", source)
    eng.load_denoiser(sd, "smpl")
    b = S.make_smpl_batch(B=B, T=T)
    eng.bind(b["cond"], T)
    betas = R.named_beta_schedule("cosine", steps)
    eng.init_diffusion(betas)
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps))
    return sd, b, R.diffusion_tables(betas), tape


def test_p_sample_teacher_forced(eng):
    """Every step of a 1000-step schedule is checked from the ORACLE's x_t (no chaotic
    amplification: see DESIGN.md 'Conditioning'), at a spread of timesteps."""
    steps = 1000
    sd, b, tables, tape = _loop_setup(eng, 4, 30, steps)
    gt, mask, cond = torch.from_numpy(b["gt"]), torch.from_numpy(b["mask"]), torch.from_numpy(b["cond"])
    model_fn = lambda x, t: R.mdm_smpl_forward(sd, x, t, cond, faithful=False)
    x = tape[0].clone()
    worst = 0.0
    for k, i in enumerate([999, 998, 750, 500, 250, 50, 2, 1, 0]):
        noise = tape[k + 1]
        with torch.no_grad():
            ref, ref0 = R.p_sample_step(model_fn, tables, x, i, noise, gt, mask)
        got, got0 = eng.p_sample(i, x.cuda(), noise.cuda(), gt.cuda(), mask.cuda())
        worst = max(worst, rel(got, ref), rel(got0, ref0))
        x = ref
    assert worst < 2e-4, worst


@pytest.mark.parametrize("use_graph", [False, True])
def test_p_sample_loop_short(eng, use_graph):
    """Full loop on an 8-step schedule, graph replay and plain launches."""
    steps = 8
    sd, b, tables, tape = _loop_setup(eng, 4, 30, steps)
    gt, mask, cond = torch.from_numpy(b["gt"]), torch.from_numpy(b["mask"]), torch.from_numpy(b["cond"])
    with torch.no_grad():
        ref = R.p_sample_loop(lambda x, t: R.mdm_smpl_forward(sd, x, t, cond, faithful=False), tables, tape, gt, mask)
    got = eng.p_sample_loop(tape.cuda(), gt.cuda(), mask.cuda(), correction=False, use_graph=use_graph).cpu()
    assert rel(got, ref) < 1e-3
    # inpainting property: the past frames of the final sample equal the ground truth exactly
    assert torch.equal(got[..., :10], gt[..., :10])


@pytest.mark.parametrize("weights", ["dense_tail", "sparse4"])
def test_smplh_lbs(eng, smplh_np, weights):
    """both skinning paths of the tensor backend: <= 8 non-zero bones per vertex (ELL list; the licensed models have
    <= 4) and the dense walk (a weight on every bone)"""
    if weights == "sparse4":
        smplh_np = S.make_smplh_model(233, sparse_weights=True)
        assert int((smplh_np["weights"] != 0).sum(1).max()) <= 4
    eng.load_body(smplh_np)
    smplh = smplh_torch(smplh_np)
    g = torch.Generator().manual_seed(1)
    Fn = 37  # not a multiple of the 16-frame skinning group
    pose = 0.4 * torch.randn(Fn, 156, generator=g)
    pose[0, 3:6] = 0
    pose[1] = 0
    betas = torch.randn(Fn, 10, generator=g)
    trans = torch.randn(Fn, 3, generator=g)
    verts, jtr = eng.lbs(pose, betas, trans)
    with torch.no_grad():
        v_ref, j_ref = R.smplh_lbs(smplh, pose, betas, trans)
    assert rel(verts, v_ref) < 1e-5 and rel(jtr, j_ref) < 1e-5
    # property: a pure translation moves every vertex by exactly that offset (to rounding)
    v2, _ = eng.lbs(pose, betas, trans + 1.0)
    assert rel(v2 - 1.0, verts) < 1e-5


def test_smplh_lbs_large_blend(eng):
    """precision budget of the tensor-core pose blend: bases 20x larger than the synthetic default (a ~10 cm corrective
    term, beyond anything the licensed model produces), large joint rotations, several row tiles of frames with a
    partial last one, an odd vertex count (unaligned output rows) - still 1e-5 of the vertex magnitude"""
    m = S.make_smplh_model(7, sparse_weights=True)
    V = 6889
    m = dict(m)
    for k in ("v_template", "shapedirs", "posedirs", "weights"):
        m[k] = np.ascontiguousarray(m[k][:V])
    m["J_regressor"] = np.ascontiguousarray(m["J_regressor"][:, :V])
    m["faces"] = np.ascontiguousarray(m["faces"][(m["faces"] < V).all(1)])
    m["posedirs"] = m["posedirs"] * 20.0
    eng.load_body(m)
    smplh = smplh_torch(m)
    g = torch.Generator().manual_seed(3)
    Fn = 300
    pose, betas, trans = 1.2 * torch.randn(Fn, 156, generator=g), 2.0 * torch.randn(Fn, 10, generator=g), torch.randn(Fn, 3, generator=g)
    verts, jtr = eng.lbs(pose, betas, trans)
    with torch.no_grad():
        v_ref, j_ref = R.smplh_lbs(smplh, pose, betas, trans)
        v64, _ = R.smplh_lbs({k: (v.double() if v.is_floating_point() else v) for k, v in smplh.items()}, pose.double(), betas.double(), trans.double())
    assert rel(verts, v_ref) < 1e-5 and rel(jtr, j_ref) < 1e-5
    # against float64 the kernel is as close as the fp32 oracle itself (within 3x)
    assert rel(verts, v64) < max(3 * rel(v_ref, v64), 2e-6)
    # the blend GEMM with TMA-multicast row-tile pairs (3 row tiles here: one pair + one tile paired with an empty one) computes
    # every element exactly like the unpaired kernel
    eng.set_gemm_multicast(False)
    v_plain, _ = eng.lbs(pose, betas, trans)
    eng.set_gemm_multicast(True)
    assert torch.equal(v_plain, verts)


def test_geometry(eng, smplh_np):
    eng.load_body(smplh_np)
    g = torch.Generator().manual_seed(2)
    verts = torch.from_numpy(smplh_np["v_template"])[None].repeat(3, 1, 1) + 0.01 * torch.randn(3, 6890, 3, generator=g)
    n = eng.vertex_normals(verts).cpu()
    n_ref = R.vertex_normals(verts, torch.from_numpy(smplh_np["faces"]))
    assert rel(n, n_ref) < 1e-5
    y = verts[:, ::13][:, :500] * 1.05 + 0.01 * torch.randn(3, 500, 3, generator=g)
    d, idx, vec = eng.signed_nn(y, verts, n_ref)
    ref = R.point2point_signed(verts, y, n_ref)
    assert torch.equal(idx.cpu().long(), ref[2])          # nearest indices: bit exact
    assert torch.equal(d.cpu().sign(), ref[0].sign())      # inside / outside decisions
    assert rel(d, ref[0]) < 1e-6 and rel(vec, ref[4]) < 1e-6
    d6 = torch.randn(1000, 6, generator=g)
    aa = eng.rot6d_to_axis_angle(d6).cpu()
    from oracle import transforms as tf
    assert rel(aa, tf.matrix_to_axis_angle(tf.rotation_6d_to_matrix(d6))) < 1e-5


def test_signed_nn_pruned_equals_brute_force(eng, smplh_np):
    """The cluster-pruned nearest-neighbour search (body-mesh targets) must reproduce the brute-force scan bit for
    bit: indices (first minimum on ties - duplicated vertices, queries sitting exactly on a vertex), signed
    distances and offset vectors; near, far and interior queries."""
    eng.load_body(smplh_np)
    g = torch.Generator().manual_seed(11)
    F = 4
    verts = torch.from_numpy(smplh_np["v_template"])[None].repeat(F, 1, 1).clone()
    verts = verts * (1.0 + 0.2 * torch.rand(F, 1, 1, generator=g)) + 0.02 * torch.randn(F, 6890, 3, generator=g)
    verts[:, 5000] = verts[:, 100]          # exact duplicates: the lower index has to win
    verts[:, 17] = verts[:, 16]
    verts[:, 6889] = verts[:, 0]
    normals = eng.vertex_normals(verts)
    q = torch.cat([verts[:, ::7] * 1.02 + 0.005 * torch.randn(F, 985, 3, generator=g),      # near the surface
                   3.0 * torch.randn(F, 300, 3, generator=g),                                # far away
                   0.1 * torch.randn(F, 200, 3, generator=g),                                # inside
                   verts[:, [100, 5000, 16, 17, 0, 6889, 3333]],                             # exactly on (duplicated) vertices
                   torch.zeros(F, 1, 3)], dim=1).contiguous()
    eng.set_nn_pruning(True)
    d1, i1, v1 = eng.signed_nn(q, verts, normals)
    eng.set_nn_pruning(False)
    d0, i0, v0 = eng.signed_nn(q, verts, normals)
    eng.set_nn_pruning(True)
    assert torch.equal(i1, i0)
    assert torch.equal(d1, d0) and torch.equal(v1, v0)
    on_vertex = i0[:, -8:-1].cpu()
    assert torch.equal(on_vertex, torch.tensor([[100, 100, 16, 16, 0, 0, 3333]] * F, dtype=torch.int32))


@pytest.mark.parametrize("source", ["random", "ref"])
def test_projector(eng, smplh_np, source):
    psd = projector_weights(source)
    eng.load_body(smplh_np)
    eng.load_projector(psd, 10, 20)
    g = torch.Generator().manual_seed(3)
    T, B = 30, 6
    ang, tr = torch.randn(T, B, 6, generator=g), torch.randn(T, B, 3, generator=g)
    hv = torch.randn(T, B, 67, 3, generator=g)
    contact = (torch.rand(B, 67, generator=g) < 0.05).long() * torch.randint(1, 5, (B, 67), generator=g)
    contact[1] = 0
    b = S.make_smpl_batch(B=B, T=T)
    eng.bind_correction(b["hand_pose"], b["betas"], b["obj_points"], past_len=10)
    got = eng.projector_sample(ang, tr, hv, contact).cpu()
    with torch.no_grad():
        ref = R.obj_projector_sample(psd, ang, tr, hv, contact, 10, 20)
    assert rel(got, ref) < 1e-4


def test_correction_hook(eng, smplh_np):
    """denoised_fn body: decisions (condition / contact) must agree exactly, continuous outputs
    within tolerance (SURVEY section 7 'discrete decisions')."""
    psd = projector_weights("auto")
    eng.load_body(smplh_np)
    eng.load_projector(psd, 10, 20)
    T, B = 30, 3
    b = S.make_smpl_batch(B=B, T=T)
    eng.bind_correction(b["hand_pose"], b["betas"], b["obj_points"], past_len=10)
    gt = torch.from_numpy(b["gt"])
    g = torch.Generator().manual_seed(4)
    x = gt + 0.02 * torch.randn(gt.shape, generator=g)
    ctx = dict(past_len=10, future_len=20, smpl_dim=132, gt=gt, hand_pose=torch.from_numpy(b["hand_pose"]),
               betas=torch.from_numpy(b["betas"]), obj_points=torch.from_numpy(b["obj_points"]),
               smplh=smplh_torch(smplh_np), projector=psd)
    with torch.no_grad():
        obs = R.correction_observables(x, ctx)
        ref = R.make_denoised_fn(ctx)(x.clone(), torch.full((B,), 450), None)
    xg = x.clone().cuda()
    got, dbg = eng.correction_apply(xg, gt.cuda(), 450, debug=True)
    assert rel(dbg["markers"], obs["markers"]) < 1e-5
    assert rel(dbg["o2h_signed"], obs["o2h_signed"]) < 1e-4
    assert torch.equal(dbg["condition"].cpu(), obs["condition"])
    assert torch.equal(dbg["contact"].cpu().long(), obs["contact"])
    assert rel(got, ref) < 1e-4


def test_full_size_properties(eng):
    """BASELINE configs[1] sizes (B=64, T=30, 100-step schedule), where the oracle takes minutes: size-independent
    properties instead.  (1) batch independence: the samples of the full batch equal the same samples denoised in
    a batch of 4 (every kernel works per row / per sample: identical on the SIMT backend; on the tensor backend the
    GEMM tile configuration and accumulator count depend on M, so equal to rounding);
    (2) the inpainted past of a sampling loop equals the ground truth exactly; (3) graph replay == eager launches,
    bit for bit; (4) two runs of the loop are bit-identical (no atomics with more than two addends anywhere)."""
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    B, T, steps = 64, 30, 100
    b = S.make_smpl_batch(B=B, T=T)
    x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0]).cuda()
    t = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(1))
    eng.bind(b["cond"], T)
    full = eng.forward(x, t.cuda()).cpu()
    pick = [0, 17, 40, 63]
    eng.bind(np.ascontiguousarray(b["cond"][:, pick]), T)
    sub = eng.forward(x[pick].contiguous(), t[pick].cuda()).cpu()
    assert rel(sub, full[pick]) < 2e-4
    eng.bind(b["cond"], T)
    eng.init_diffusion(R.named_beta_schedule("cosine", steps))
    tape = torch.from_numpy(S.noise_tape(b["gt"].shape, steps)).cuda()
    gt, mask = torch.from_numpy(b["gt"]).cuda(), torch.from_numpy(b["mask"]).cuda()
    a1 = eng.p_sample_loop(tape, gt, mask, use_graph=True).clone()
    a2 = eng.p_sample_loop(tape, gt, mask, use_graph=True).clone()
    a3 = eng.p_sample_loop(tape, gt, mask, use_graph=False).clone()
    assert torch.equal(a1, a2) and torch.equal(a1, a3)
    assert torch.equal(a1[mask], gt[mask])
    assert torch.isfinite(a1).all()


@pytest.mark.parametrize("M", [1920, 129])
def test_fused_feed_forward_with_final_norm(eng, M):
    """level 2 of the fused feed-forward kernel: the layer's final LayerNorm applied in the reduction epilogue (two
    named barriers across the 256 reducing threads), against float64 - and a whole forward with it switched on."""
    g = torch.Generator().manual_seed(M + 1)
    x = torch.randn(M, 256, generator=g)
    w1 = torch.randn(1024, 256, generator=g) / 16
    b1 = torch.randn(1024, generator=g) * 0.1
    w2 = torch.randn(256, 1024, generator=g) / 32
    b2 = torch.randn(256, generator=g) * 0.1
    res = torch.randn(M, 256, generator=g)
    lw, lb = 1.0 + 0.1 * torch.randn(256, generator=g), 0.1 * torch.randn(256, generator=g)
    ref = torch.nn.functional.gelu(x.double() @ w1.double().T + b1.double()) @ w2.double().T + b2.double() + res.double()
    want = torch.nn.functional.layer_norm(ref, (256,), lw.double(), lb.double(), 1e-5)
    got = eng.mlp(x, w1, b1, w2, b2, res, ln_w=lw, ln_b=lb).cpu().double()
    assert ((got - want).abs().max() / want.abs().max()).item() < 5e-6
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    b = S.make_smpl_batch(B=4, T=30)
    eng.bind(b["cond"], 30)
    xx = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0])
    t = torch.tensor([900, 400, 50, 0])
    with torch.no_grad():
        ref_out = R.mdm_smpl_forward(sd, xx, t, torch.from_numpy(b["cond"]), faithful=False)
    outs = {}
    for level in (1, 2, 3):    # 1 = feed-forward only (the norm stays with the next kernel), 2 = default, 3 = whole layer in one launch
        eng.set_fused_mlp(level)
        outs[level] = eng.forward(xx.cuda(), t.cuda()).cpu()
        assert rel(outs[level], ref_out) < 2e-4, level
    eng.set_fused_mlp(2)
    if M == 1920:
        # level 3 (attention + feed-forward of a layer in ONE cluster kernel on sample-aligned 4-sample tiles) computes every
        # row exactly like level 2: bit-identical, also with a partial last cluster (B = 7) and a 3-slab window (T = 35)
        assert torch.equal(outs[3], outs[2])
        for B2, T2 in ((7, 30), (3, 35), (9, 16)):
            b2 = S.make_smpl_batch(B=B2, T=T2)
            eng.bind(b2["cond"], T2)
            x2 = torch.from_numpy(S.noise_tape(b2["gt"].shape, 0)[0]).cuda()
            t2 = torch.randint(0, 1000, (B2,), generator=torch.Generator().manual_seed(B2)).cuda()
            o = {}
            for level in (2, 3):
                eng.set_fused_mlp(level)
                o[level] = eng.forward(x2, t2).clone()
            eng.set_fused_mlp(2)
            assert torch.equal(o[2], o[3]), (B2, T2)


def test_launch_structure_switches_bit_identical(eng):
    """The launch-structure options of the step compute every row with the same arithmetic: self- + cross-attention of the
    standard layers as one launch vs two (idb_set_fused_mlp 11 / 10), 128- vs 64-column GEMM tiles
    (idb_debug_set_gemm_accumulators 901 / 900; the hook keeps its name, other values set the fp32 promotion interval:
    same operations in the same k order per element whatever the tile width)."""
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    for B2, T2 in ((64, 30), (5, 35), (9, 16)):
        b = S.make_smpl_batch(B=B2, T=T2)
        eng.bind(b["cond"], T2)
        x = torch.from_numpy(S.noise_tape(b["gt"].shape, 0)[0]).cuda()
        t = torch.randint(0, 1000, (B2,), generator=torch.Generator().manual_seed(B2)).cuda()
        base = eng.forward(x, t).clone()
        eng.set_fused_mlp(10)
        two = eng.forward(x, t).clone()
        eng.set_fused_mlp(11)
        eng.lib.idb_debug_set_gemm_accumulators(900)
        eng.set_fused_mlp(2)          # (drops the captured graphs)
        wide = eng.forward(x, t).clone()
        eng.lib.idb_debug_set_gemm_accumulators(901)
        eng.set_fused_mlp(2)
        assert torch.equal(base, two), (B2, T2)
        assert torch.equal(base, wide), (B2, T2)


def test_rotation_conversions_targeted(eng):
    """A11: the 6D -> axis-angle chain (rotation_6d_to_matrix -> matrix_to_quaternion's 4-candidate argmax -> axis-angle with the
    small-angle series) on the cases random inputs do not reach: rotations within 1e-3 .. 1e-6 of pi (where the argmax
    switches between the x / y / z candidates), exact 180-degree turns about the axes, near-identity rotations on both sides
    of the 1e-6 series switch, un-normalised and nearly collinear 6D inputs.  Near pi the axis-angle vector itself is
    ill-conditioned (aa and -aa describe almost the same rotation), so the comparison is made on the rotation matrices the
    two results describe; away from pi the vectors are compared directly."""
    from oracle import transforms as tf
    g = torch.Generator().manual_seed(17)
    axes = torch.nn.functional.normalize(torch.randn(64, 3, generator=g), dim=1)
    axes = torch.cat([axes, torch.eye(3), -torch.eye(3), torch.tensor([[0.7071068, 0.7071068, 0.0], [0.0, 0.7071068, -0.7071068]])])
    angles = torch.tensor([3.14159265, 3.1415, 3.1406, 3.1316, 3.0416, 1e-7, 9e-7, 1.1e-6, 1e-5, 1e-3, 0.0, 1.5707963])
    aa = (axes[:, None, :] * angles[None, :, None]).reshape(-1, 3)
    Rm = tf.axis_angle_to_matrix(aa.double()).float()
    d6 = tf.matrix_to_rotation_6d(Rm)
    d6 = torch.cat([d6, d6 * torch.tensor([3.0, 3.0, 3.0, 0.2, 0.2, 0.2]),                       # un-normalised rows
                    torch.cat([d6[:, :3], d6[:, :3] + 0.05 * d6[:, 3:]], dim=1)])                  # second row close to the first (Gram-Schmidt cancels 20x)
    got = eng.rot6d_to_axis_angle(d6).cpu()
    want = tf.matrix_to_axis_angle(tf.rotation_6d_to_matrix(d6))
    R_got, R_want = tf.axis_angle_to_matrix(got), tf.axis_angle_to_matrix(want)
    assert torch.isfinite(got).all()
    assert (R_got - R_want).abs().max().item() < 5e-5, (R_got - R_want).abs().max().item()
    far = (want.norm(dim=1) < 3.0)                 # well away from pi: the vectors themselves agree
    assert rel(got[far], want[far]) < 5e-5, rel(got[far], want[far])
