"""The deformation's Jacobian (nsb_deform_jacobian) and inverse (nsb_deform_inverse) on the GPU, point tracking and mesh
sequences: J against the CPU oracle and the input-gradient kernel, a rigid warp with a known inverse, Newton on random
heads against the float64 oracle, the damping rule, tile edges and repeatability, two timesteps that differ by a rotation,
and the model methods.  Heads are drawn from U(+-2e-2) as in test_gpu_deform_jacobian.py: fresh U(+-1e-5) heads would
make J ~ 0 and prove nothing."""
import os

import numpy as np
import pytest
import torch

from conftest import native_from_oracle, oracle_params
from deform_inverse_oracle import as_float64, jacobian_by_pullbacks, newton_inverse, rigid_inverse, rigid_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = dict(seed=19980801, n_timesteps=24, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
             deform_last_scale=2e-2)      # non-cubic default box: a misplaced D^-1 fails
WD = 7.0


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@pytest.fixture(scope="module")
def deformed():
    P = oracle_params(KNOBS)
    return P, native_from_oracle(P, DEV)


def _points(P, n, seed, margin=0.0):
    gen = torch.Generator().manual_seed(seed)
    pos = P.aabb[0] + (margin + (1 - 2 * margin) * torch.rand((n, 3), generator=gen)) * (P.aabb[1] - P.aabb[0])
    return pos, torch.rand((n,), generator=gen), gen


def _row_errors(got, want):
    """relative L2 per row of J ([n,3,3] -> [3n])"""
    g, w = got.reshape(-1, 3), want.reshape(-1, 3)
    return (g - w).norm(dim=-1) / w.norm(dim=-1).clamp_min(1e-20)


def _check_rows(got, want, what):
    rel = _row_errors(got, want)
    n_off = int((rel > 2e-2).sum())
    print(f"{what}: {n_off} of {rel.numel()} rows above 2e-2, worst {rel.max().item():.3e}")
    assert n_off <= 0.001 * rel.numel(), (what, n_off, rel.numel(), rel.max().item())


@pytest.mark.parametrize("window", [None, 3.5])
def test_jacobian_matches_the_oracle_table_codes(deformed, window):
    from nersemble_b200 import ops
    P, NP = deformed
    pos, times, _ = _points(P, 3000, 1, margin=-0.03)
    wc = P.time_emb_deform[pl.timesteps_from_times(times, P.n_timesteps)]
    got = ops.deform_jacobian(NP, window_deform=window, positions=pos.to(DEV), sample_times=times.to(DEV))
    want = jacobian_by_pullbacks(P, pos, wc, window)
    assert (want.norm(dim=(-2, -1)) >= 0.1).float().mean() > 0.9
    _check_rows(got["jacobian"].cpu(), want, f"J, table codes, window {window}")
    # the existing input-gradient kernel's J^T e_i is row i of J
    for i in range(3):
        u = torch.zeros((pos.shape[0], 3), device=DEV); u[:, i] = 1.0
        jt = ops.deform_input_grad(NP, u, window_deform=window, positions=pos.to(DEV), sample_times=times.to(DEV)).cpu()
        _check_rows(got["jacobian"].cpu()[:, i], jt, f"J row {i} against J^T e_{i}")
    # offsets: the same stem as field_forward's deformation role up to fp16 operand rounding and fp32 summation order
    ff = ops.field_forward(NP, window_deform=window, positions=pos.to(DEV), sample_times=times.to(DEV), want=("offsets",))
    d = (got["offsets"] - ff["offsets"]).abs()
    print(f"offsets vs field_forward: max {d.max().item():.3e}, 99.9 % {d.amax(-1).quantile(0.999).item():.3e}")
    assert d.max().item() <= 2e-4, d.max().item()


@pytest.mark.parametrize("window", [None, 3.5])
def test_jacobian_matches_the_oracle_per_sample_codes(deformed, window):
    from nersemble_b200 import ops
    P, NP = deformed
    pos, _, gen = _points(P, 3000, 7, margin=-0.05)
    wc = torch.randn((pos.shape[0], 128), generator=gen) * 0.1
    got = ops.deform_jacobian(NP, window_deform=window, positions=pos.to(DEV), sample_warp_codes=wc.to(DEV))
    want = jacobian_by_pullbacks(P, pos, wc.half().float(), window)
    assert (want.norm(dim=(-2, -1)) >= 0.1).float().mean() > 0.9
    _check_rows(got["jacobian"].cpu(), want, f"J, per-sample codes, window {window}")
    ff = ops.field_forward(NP, window_deform=window, positions=pos.to(DEV), sample_warp_codes=wc.to(DEV), want=("offsets",))
    assert (got["offsets"] - ff["offsets"]).abs().max().item() <= 2e-4


@pytest.mark.parametrize("r", [(0.1, -0.15, 0.12), (3e-3, -2e-3, 1e-3)], ids=["rotation", "clamped_theta"])
def test_rigid_warp_inverse_is_the_analytic_one(r):
    from nersemble_b200 import ops
    v = (0.02, -0.03, 0.01)
    P = rigid_params(r, v)
    NP = native_from_oracle(P, DEV)
    gen = torch.Generator().manual_seed(3)
    n = 3000
    c = 0.3 + 0.4 * torch.rand((n, 3), generator=gen)
    times = torch.rand((n,), generator=gen)
    out = ops.deform_inverse(NP, c.to(DEV), sample_times=times.to(DEV), window_deform=WD)
    P64 = as_float64(P)
    want = rigid_inverse(c.double(), P64.r_b, P64.v_b)
    err = (out["positions"].cpu().double() - want).abs().max().item()
    print(f"rigid {r}: max error {err:.3e}, iterations max {int(out['iterations'].max())}")
    assert bool(out["converged"].all()) and err <= 1e-5, err
    jac = ops.deform_jacobian(NP, window_deform=WD, positions=c.to(DEV), sample_times=times.to(DEV))["jacobian"].cpu()
    th = torch.tensor(r).norm()
    K = torch.tensor([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    R = torch.eye(3) + (th.sin() / th) * K + ((1 - th.cos()) / th ** 2) * (K @ K) if th * th > 1e-4 else None
    if R is not None:
        assert (jac - (R - torch.eye(3))).abs().max().item() <= 1e-5


def _residual(NP, pos, targets, off):
    """|F|inf of the kernels' own formula: box_coord(p + offset) - box_coord(c)."""
    lo = torch.tensor(NP.aabb_list[:3], device=pos.device)
    ext = torch.tensor(NP.aabb_list[3:], device=pos.device) - lo
    return (((pos + off) - lo) / ext - (targets - lo) / ext).abs().amax(-1)


def test_random_heads_converge_and_agree_with_the_float64_oracle(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    pos, times, _ = _points(P, 4000, 21, margin=0.05)
    pd, td = pos.to(DEV), times.to(DEV)
    targets = pd + ops.field_forward(NP, window_deform=WD, positions=pd, sample_times=td, want=("offsets",))["offsets"]
    out = ops.deform_inverse(NP, targets, sample_times=td, window_deform=WD, tol=1e-4)
    conv = out["converged"]
    hist = torch.bincount(out["iterations"].long().cpu(), minlength=21)
    print(f"random heads: {conv.float().mean().item():.5f} converged, iterations {hist.tolist()}")
    assert conv.float().mean().item() >= 0.999
    # re-evaluated with the Jacobian mode: within tol
    p = out["positions"]
    off_j = ops.deform_jacobian(NP, window_deform=WD, positions=p, sample_times=td)["offsets"]
    assert (_residual(NP, p, targets, off_j)[conv] <= 1e-4 * (1 + 1e-3)).all()
    assert torch.equal(out["residual"][conv] < 1e-4, torch.ones_like(conv[conv]))
    # against field_forward's own warp: within tol plus the measured gap between the two roles (D^-1 x 2e-4 at most)
    off_f = ops.field_forward(NP, window_deform=WD, positions=p, sample_times=td, want=("offsets",))["offsets"]
    gap = (off_f - off_j).abs().max().item() / min(NP.aabb_list[3 + k] - NP.aabb_list[k] for k in range(3))
    rf = _residual(NP, p, targets, off_f)[conv]
    print(f"residual through field_forward: max {rf.max().item():.3e} (role gap {gap:.3e})")
    assert (rf <= 1e-4 + gap + 1e-6).all()
    # the float64 oracle's solution of the same targets (kernel-precision J, float64 Newton): the roots differ by the
    # fp16 rounding of the warp, |dp_n| <~ |(I + D^-1 J)^-1| (tol + rounding gap)
    sel = torch.arange(0, 4000, 10)
    Precision.mode = "none"
    P64 = as_float64(P)
    wc = P.time_emb_deform[pl.timesteps_from_times(times[sel], P.n_timesteps)]
    want, res64 = newton_inverse(P64, targets.cpu()[sel].double(), wc, WD, init=None)
    Precision.mode = "kernel"
    ext = (P.aabb[1] - P.aabb[0]).double()
    err = ((out["positions"].cpu()[sel].double() - want) / ext).abs().amax(-1)
    ok = conv.cpu()[sel] & (res64 < 1e-12)
    print(f"against the float64 oracle: median {err[ok].median().item():.3e}, max {err[ok].max().item():.3e} (normalised)")
    assert ok.float().mean() > 0.99 and err[ok].max().item() <= 2e-3 and err[ok].median().item() <= 2e-4


def test_damping_never_returns_a_worse_point(deformed):
    """Heads ten times stronger (rotations of up to ~1 rad from one point to the next): undamped Newton overshoots.  No
    returned residual exceeds the initial one, and exactly the points whose residual is not below tol are flagged."""
    from nersemble_b200 import ops
    P0, _ = deformed
    import copy
    P = copy.deepcopy(P0)
    P.r_w.mul_(10.0); P.v_w.mul_(10.0)
    NP = native_from_oracle(P, DEV)
    pos, times, _ = _points(P, 4000, 5, margin=0.05)
    pd, td = pos.to(DEV), times.to(DEV)
    targets = pd + ops.field_forward(NP, window_deform=WD, positions=pd, sample_times=td, want=("offsets",))["offsets"]
    out = ops.deform_inverse(NP, targets, sample_times=td, window_deform=WD, max_iter=12)
    off0 = ops.deform_jacobian(NP, window_deform=WD, positions=targets, sample_times=td)["offsets"]
    r0 = _residual(NP, targets, targets, off0)
    hist = torch.bincount(out["iterations"].long().cpu(), minlength=13)
    print(f"strong heads: {out['converged'].float().mean().item():.4f} converged, status {torch.bincount(out['status'].long().cpu()).tolist()}, "
          f"iterations {hist.tolist()}, initial residual median {r0.median().item():.3e}")
    assert (out["residual"] <= r0).all()
    assert torch.equal(out["converged"], out["residual"] < 1e-4)
    assert ((out["status"] == 0) | (out["status"] == 1) | (out["status"] == 2)).all()
    assert (out["iterations"][~out["converged"] & (out["status"] == 1)] == 12).all()
    assert (r0 >= 1e-2).float().mean() > 0.5           # the initial guesses are far off


def test_edges_repeatability_and_tracking_to_the_source_time(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    pos, times, _ = _points(P, 4097, 9, margin=0.05)
    pd, td = pos.to(DEV), times.to(DEV)
    targets = pd + ops.deform_jacobian(NP, window_deform=WD, positions=pd, sample_times=td)["offsets"]
    full = ops.deform_inverse(NP, targets, sample_times=td, window_deform=WD)
    again = ops.deform_inverse(NP, targets, sample_times=td, window_deform=WD)
    jf = ops.deform_jacobian(NP, window_deform=WD, positions=pd, sample_times=td)
    jg = ops.deform_jacobian(NP, window_deform=WD, positions=pd, sample_times=td)
    for k in full:
        assert torch.equal(full[k], again[k]), k
    assert torch.equal(jf["jacobian"], jg["jacobian"]) and torch.equal(jf["offsets"], jg["offsets"])
    for n in (0, 1, 31, 32, 33):
        part = ops.deform_inverse(NP, targets[:n], sample_times=td[:n], window_deform=WD)
        for k in full:
            assert torch.equal(part[k], full[k][:n]), (n, k)
        pj = ops.deform_jacobian(NP, window_deform=WD, positions=pd[:n], sample_times=td[:n])
        assert torch.equal(pj["jacobian"], jf["jacobian"][:n]) and pj["jacobian"].shape == (n, 3, 3)
    # tracking to the source time: the points come back bit for bit, with 0 iterations
    t0 = 5.0 / 23.0
    tr = ops.track_points(NP, pd, time_from=t0, times_to=[t0, 9.0 / 23.0], window_deform=WD)
    assert torch.equal(tr["positions"][0], pd) and (tr["iterations"][0] == 0).all() and tr["converged"][0].all()
    assert tr["converged"][1].float().mean() >= 0.999 and not torch.equal(tr["positions"][1], pd)


def _rotation(r):
    th = (r * r).sum().clamp_min(1e-4).sqrt()
    K = torch.tensor([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    return torch.eye(3) + (th.sin() / th) * K + ((1 - th.cos()) / th ** 2) * (K @ K)


def _two_frame_params():
    """The fixture of test_rotation_between_two_timesteps_turns_the_observation_normals: timestep 0 the identity,
    timestep 1 a rotation R about the box origin (unit-cube box), one geometry; here with a smooth field (levels of
    resolution <= 33) that a 64^3 grid resolves."""
    r = torch.tensor([0.0625, -0.125, 0.25])
    P = rigid_params((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    P.deform_w[0][0, 45] = 1.0
    for l in (1, 2, 3, 5):
        P.deform_w[l][0, 0] = 1.0
    P.deform_w[4][0, 173] = 1.0
    P.r_w.zero_(); P.v_w.zero_(); P.r_w[:, 0] = r
    P.time_emb_deform.zero_(); P.time_emb_deform[1, 0] = 1.0
    P.time_emb[1] = P.time_emb[0]
    P.tables[int(P.levels.offset[3]):] = 0
    return P, _rotation(r)


def _nearest_distance(a, b):
    a, b = a.to(DEV), b.to(DEV)
    return torch.cat([torch.cdist(a[i:i + 2048], b).min(1).values for i in range(0, a.shape[0], 2048)]).cpu()


def test_rotation_between_two_timesteps_tracks_points_and_meshes():
    from nersemble_b200 import ops
    P, Rm = _two_frame_params()
    NP = native_from_oracle(P, DEV)
    gen = torch.Generator().manual_seed(13)
    p0 = (0.35 + 0.3 * torch.rand((2000, 3), generator=gen)).to(DEV)
    tr = ops.track_points(NP, p0, time_from=0.0, times_to=[1.0], window_deform=WD)
    Rd = Rm.to(DEV)
    err = (tr["positions"][0] - p0 @ Rd).abs().max().item()      # rows: R^T p0
    print(f"tracked points vs R^T p: {err:.3e}")
    assert tr["converged"].all() and err <= 1e-5
    WH = 32.0
    can_g = ops.density_grid(NP, time=0.0, resolution=64, space="canonical", window_hash=WH)["sigma"]
    level = float(can_g[16:48, 16:48, 16:48].median())
    seq = ops.extract_mesh_sequence(NP, times=[0.0, 1.0], reference_time=0.0, level=level, resolution=64,
                                    window_hash=WH, window_deform=WD)
    v0, v1 = seq["vertices"][0], seq["vertices"][1]
    ref = ops.extract_mesh(NP, time=0.0, level=level, resolution=64, window_hash=WH, window_deform=WD)
    assert torch.equal(v0, ref["vertices"]) and torch.equal(seq["faces"], ref["faces"])
    assert torch.equal(seq["normals"][0], ref["normals"]) and torch.equal(seq["colours"][0], ref["colours"])
    assert seq["converged"].all()
    assert (v1 - v0 @ Rd).abs().max().item() <= 1e-5
    # against frame 1's own mesh: Chamfer below one voxel over the interior
    own = ops.extract_mesh(NP, time=1.0, level=level, resolution=64, window_hash=WH, window_deform=WD,
                           normals=False, colours=False)["vertices"]
    voxel = 1.0 / 63
    inner = lambda p: ((p > 0.3) & (p < 0.7)).all(-1)
    a, b = v1[inner(v1)].cpu(), own[inner(own)].cpu()
    assert a.shape[0] > 500 and b.shape[0] > 500
    chamfer = 0.5 * (_nearest_distance(a, own.cpu()).mean() + _nearest_distance(b, v1.cpu()).mean())
    print(f"tracked frame 1 vs its own mesh: chamfer {chamfer / voxel:.3f} voxel")
    assert chamfer < voxel
    # sigma at the tracked vertices: the same canonical points, so the level up to the grid interpolation of frame 0
    s0, s1 = seq["sigma"][0], seq["sigma"][1]
    dev0 = ((s0 - level).abs() / level).median().item()
    print(f"sigma: frame 0 median |s/level - 1| {dev0:.3e}, frames 0 / 1 max relative difference "
          f"{((s1 - s0).abs() / s0.abs().clamp_min(1e-6)).max().item():.3e}")
    assert dev0 <= 0.1
    assert ((s1 - s0).abs() <= 1e-2 * s0.abs() + 1e-3 * level).float().mean() >= 0.99
    # normals turn with the head: n1 = R^T n0 where both warped positions are inside the box
    n0, n1 = seq["normals"][0], seq["normals"][1]
    both = (n0.norm(dim=-1) > 0) & (n1.norm(dim=-1) > 0)
    cos = (n1[both] * (n0[both] @ Rd)).sum(-1)
    print(f"normals: median cos {cos.median().item():.6f}, {(cos > 0.999).float().mean().item():.4f} above 0.999")
    assert both.float().mean() > 0.9 and cos.median() > 0.9999 and (cos > 0.999).float().mean() > 0.99


@pytest.mark.parametrize("deform", [True, False])
def test_model_track_points_and_mesh_sequence(tmp_path, deform):
    from nersemble_b200.mesh import Mesh, MeshSequence
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P = oracle_params(dict(KNOBS, n_timesteps=4))
    m = make_model(T=4, log2T=14)
    load_oracle_params_into(m, P)
    m.config.use_deformation_field = deform       # without it the model renders, meshes and tracks undeformed
    m = m.to(DEV).eval()
    m.occupancy_grid.binaries[0] = blob_grid(5).to(DEV)
    pts = (P.aabb[0] + torch.rand((100, 3), generator=torch.Generator().manual_seed(4)) * (P.aabb[1] - P.aabb[0])).to(DEV)
    tr = m.track_points(pts, 1, [0, 1, 3])
    assert tr["positions"].shape == (3, 100, 3) and tr["converged"].shape == (3, 100)
    assert torch.equal(tr["positions"][1], pts)
    if deform:
        assert tr["converged"].float().mean() > 0.99 and not torch.equal(tr["positions"][0], pts)
    else:
        assert all(torch.equal(tr["positions"][i], pts) for i in range(3)) and tr["converged"].all()
    from nersemble_b200 import ops
    wh, wd = m._windows()
    g = ops.density_grid(m.native_params(), time=2.0 / 3.0, resolution=24, window_hash=wh, window_deform=wd, **m._blend_opts())
    level = float(g["sigma"][1:-1, 1:-1, 1:-1].median())
    seq = m.extract_mesh_sequence([0, 2, 3], reference_timestep=2, resolution=24, level=level, respect_occupancy=False)
    assert isinstance(seq, MeshSequence) and len(seq) == 3 and seq.timesteps == [0, 2, 3]
    V = seq.vertices.shape[1]
    assert V > 100 and seq.vertices.shape == (3, V, 3) and seq.normals.shape == (3, V, 3) and seq.colours.shape == (3, V, 3)
    assert seq.sigma.shape == (3, V) and seq.converged.dtype == bool and seq.converged.mean() > 0.99
    ref = m.extract_mesh(2, resolution=24, level=level, respect_occupancy=False)
    assert np.array_equal(seq.faces, ref.faces) and np.array_equal(seq.vertices[1], ref.vertices)
    paths = seq.save_ply(str(tmp_path / "head_{:02d}.ply"))
    assert [os.path.basename(p) for p in paths] == ["head_00.ply", "head_02.ply", "head_03.ply"]
    for i, p in enumerate(paths):
        back = Mesh.load_ply(p)
        assert np.array_equal(back.vertices, seq.vertices[i]) and np.array_equal(back.faces, seq.faces)
