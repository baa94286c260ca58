"""Rendering between captured timesteps (time_interpolation="linear", DESIGN 4.2g) on the GPU: bit-identity with the
nearest path at integer times (uniform frame, timestep stack, line gather, both samplers); a uniform fractional time
against a model whose embeddings hold the interpolated codes as an extra row and against the float64 oracle; mixed
fractional times against per-ray uniform renders and the per-sample-code path; continuity at the snap boundary;
determinism and no host synchronisation; the model attribute."""
import copy

import pytest
import torch

from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
             deform_last_scale=1e-3)
WH, WD = 32.0, 7.0
RGB_L2 = 1e-3       # per-ray RGB L2, accumulation and depth: the tolerances of DESIGN 5 between two gather paths


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@pytest.fixture(scope="module")
def trained():
    P = oracle_params(KNOBS)
    return P, native_from_oracle(P, DEV)


def _rays(R, seed):
    from oracle.gen_golden import ring_rays
    o, d, t, _ = ring_rays(R, seed)
    return o.to(DEV), d.to(DEV), t.to(DEV)


def _render(NP, o, d, t, sampler="fixed", **kw):
    from nersemble_b200 import ops
    if sampler == "fixed":
        return ops.render_rays(NP, o, d, t, window_hash=WH, window_deform=WD, sampler="fixed", n_per_ray=50,
                               near_plane=0.2, step=0.011, **kw)
    from oracle.gen_golden import blob_grid
    R = o.shape[0]
    aabb = torch.tensor([float(v) for v in NP.aabb_list], device=DEV).reshape(1, 6)
    return ops.render_rays(NP, o, d, t, window_hash=WH, window_deform=WD, sampler="occupancy",
                           near_planes=torch.full((R,), 0.2, device=DEV), far_planes=torch.full((R,), 1e3, device=DEV),
                           binaries=blob_grid(5)[None].to(DEV), aabbs=aabb, step=0.011, capacity=R * 600, **kw)


def _equal(a, b, what=""):
    for k in ("rgb", "accumulation", "depth", "deformation", "packed_info"):
        assert torch.equal(a[k], b[k]), (what, k)
    pa, pb = a.packed(), b.packed()
    for k in ("t_starts", "sigma", "rgb", "offsets", "weights"):
        assert torch.equal(pa[k], pb[k]), (what, k)


def _close(a, b, what="", l2=RGB_L2):
    err = (a["rgb"] - b["rgb"]).norm(dim=-1).max().item()
    assert err < l2, (what, err)
    torch.testing.assert_close(a["accumulation"], b["accumulation"], rtol=0, atol=RGB_L2)
    torch.testing.assert_close(a["depth"], b["depth"], rtol=RGB_L2, atol=RGB_L2)
    return err


def _extra_row(P, t):
    """The oracle parameters with the codes at time t (time_lerp of the fp32 rows) appended as timestep T: a nearest
    render of that model at t = 1 evaluates the field at the interpolated codes."""
    from nersemble_b200 import ops
    T = P.time_emb.shape[0]
    i0, i1, lam = ops.time_lerp(t, T)
    Q = copy.copy(P)
    Q.time_emb = torch.cat([P.time_emb, ops._lerp_f32(P.time_emb[i0:i0 + 1].float(), P.time_emb[i1:i1 + 1].float(), lam)])
    wd = P.time_emb_deform.half().float()         # NativeParams keeps the warp codes in fp16
    Q.time_emb_deform = torch.cat([P.time_emb_deform, ops._lerp_f32(wd[i0:i0 + 1], wd[i1:i1 + 1], lam)])
    return Q


@pytest.mark.parametrize("sampler", ["fixed", "occupancy"])
def test_integer_times_are_the_nearest_render_bit_for_bit(trained, sampler):
    _, NP = trained
    T = NP.n_timesteps
    o, d, _ = _rays(48, 3)
    k = torch.randint(0, T, (48, 1), generator=torch.Generator().manual_seed(0)).to(DEV)
    t = k.float() / (T - 1)
    for line in (False, True):          # the timestep stack and the line gather
        _equal(_render(NP, o, d, t, sampler, line_gather=line, time_interpolation="linear"),
               _render(NP, o, d, t, sampler, line_gather=line), f"mixed line={line}")
    for j in range(T):                  # the uniform frame on the at_time view
        tj = torch.full_like(t, j / (T - 1))
        _equal(_render(NP, o, d, tj, sampler, uniform_time=j / (T - 1), time_interpolation="linear"),
               _render(NP, o, d, tj, sampler, uniform_time=j / (T - 1)), f"uniform {j}")


def test_integer_times_bit_for_bit_with_40_timesteps():
    P = oracle_params(dict(KNOBS, n_timesteps=40))
    NP = native_from_oracle(P, DEV)
    assert NP.timestep_tables(WH, True, True) is None             # T > 32: the line gather
    o, d, _ = _rays(40, 4)
    t = (torch.arange(40, device=DEV).float() / 39)[:, None]
    _equal(_render(NP, o, d, t, time_interpolation="linear"), _render(NP, o, d, t), "T=40")


def test_uniform_fractional_time_matches_the_extra_row_model_and_the_mixed_kernels(trained):
    P, NP = trained
    o, d, _ = _rays(60, 5)
    for t in (0.2, 0.55, 0.9):
        NQ = native_from_oracle(_extra_row(P, t), DEV)
        tt = torch.full((60, 1), t, device=DEV)
        lin = _render(NP, o, d, tt, uniform_time=t, time_interpolation="linear")
        ref = _render(NQ, o, d, torch.ones_like(tt), uniform_time=1.0)
        _close(lin, ref, f"extra row t={t}")
        torch.testing.assert_close(lin["deformation"], ref["deformation"], rtol=0, atol=1e-5)
        for line in (False, True):
            _close(_render(NP, o, d, tt, line_gather=line, time_interpolation="linear"), lin, f"mixed t={t} line={line}")


def test_uniform_fractional_time_against_the_float64_oracle(trained):
    from nersemble_b200 import ops
    P, NP = trained
    R, t = 40, 0.45
    o, d, _ = _rays(R, 6)
    ts, te, ri = pl.fixed_samples(o.cpu(), d.cpu(), P.aabb, 50, 0.011, near=0.2)
    Q = _extra_row(P, t)
    with torch.no_grad():
        want = pl.render(Q, o.cpu(), d.cpu(), torch.ones((R, 1)), ts, te, ri, window_hash=WH, window_deform=WD, training=False)
    tt = torch.full((R, 1), t, device=DEV)
    for kw in (dict(uniform_time=t), dict(), dict(line_gather=True)):
        got = _render(NP, o, d, tt, time_interpolation="linear", **kw)
        err = (got["rgb"].cpu() - want["rgb"]).norm(dim=-1).max().item()
        print(f"float64 oracle {kw}: max per-ray RGB L2 {err:.3e}")
        assert err < 1e-3, (kw, err)


@pytest.mark.parametrize("line", [False, True])
def test_mixed_fractional_times(trained, line):
    from nersemble_b200 import ops
    P, NP = trained
    R = 32
    o, d, _ = _rays(R, 7)
    t = torch.rand((R, 1), generator=torch.Generator().manual_seed(3)).to(DEV)
    mixed = _render(NP, o, d, t, line_gather=line, time_interpolation="linear")
    near = _render(NP, o, d, t, line_gather=line)
    assert torch.equal(mixed["num_samples_per_ray"], near["num_samples_per_ray"])
    # each ray against a uniform render at its own time
    worst = 0.0
    for r in range(R):
        one = _render(NP, o[r:r + 1], d[r:r + 1], t[r:r + 1], uniform_time=float(t[r]), time_interpolation="linear")
        worst = max(worst, (one["rgb"][0] - mixed["rgb"][r]).norm().item())
        torch.testing.assert_close(one["depth"][0], mixed["depth"][r], rtol=RGB_L2, atol=RGB_L2)
    print(f"mixed vs per-ray uniform (line={line}): max per-ray RGB L2 {worst:.3e}")
    assert worst < RGB_L2
    # against the per-sample-code kernels on the render's own packed samples
    pk = mixed.packed()
    codes = ops.time_codes(NP, t)
    ri = pk["ray_indices"].long()
    f = ops.field_forward(NP, origins=o, directions=d, ray_times=t.reshape(-1), t_starts=pk["t_starts"], t_ends=pk["t_ends"],
                          ray_indices=pk["ray_indices"], window_hash=WH, window_deform=WD,
                          sample_blend_codes=codes["blend_codes"][ri].contiguous(),
                          sample_warp_codes=codes["warp_codes"][ri].contiguous())
    c = ops.composite(mixed["packed_info"], pk["t_starts"], pk["t_ends"], f["sigma"], f["rgb"], f["offsets"])
    err = _close(mixed, c, "per-sample codes")
    print(f"mixed vs per-sample codes (line={line}): max per-ray RGB L2 {err:.3e}")


def test_continuity_at_the_snap_boundary(trained):
    _, NP = trained
    T = NP.n_timesteps
    o, d, _ = _rays(48, 8)
    k = 2
    base = _render(NP, o, d, torch.full((48, 1), k / (T - 1), device=DEV), time_interpolation="linear")
    step = _render(NP, o, d, torch.full((48, 1), (k + 1) / (T - 1), device=DEV), time_interpolation="linear")
    jump = (step["rgb"] - base["rgb"]).norm(dim=-1).max().item()
    for du in (0.5 * 2 ** -10, -0.5 * 2 ** -10):          # inside the snap: the integer render bit for bit
        got = _render(NP, o, d, torch.full((48, 1), (k + du) / (T - 1), device=DEV), time_interpolation="linear")
        assert torch.equal(got["rgb"], base["rgb"])
    for du in (2 ** -9, -2 ** -9, 4e-3):                  # just outside: within |du| of one timestep's change
        got = _render(NP, o, d, torch.full((48, 1), (k + du) / (T - 1), device=DEV), time_interpolation="linear")
        err = (got["rgb"] - base["rgb"]).norm(dim=-1).max().item()
        assert err <= 4 * abs(du) * jump + RGB_L2, (du, err, jump)


def test_deterministic_and_free_of_host_synchronisation(trained):
    _, NP = trained
    o, d, _ = _rays(64, 9)
    t = torch.rand((64, 1), generator=torch.Generator().manual_seed(4)).to(DEV)
    first = {line: _render(NP, o, d, t, line_gather=line, time_interpolation="linear") for line in (False, True)}
    uni = _render(NP, o, d, torch.full_like(t, 0.3), uniform_time=0.3, time_interpolation="linear")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = {line: _render(NP, o, d, t, line_gather=line, time_interpolation="linear") for line in (False, True)}
        uni2 = _render(NP, o, d, torch.full_like(t, 0.3), uniform_time=0.3, time_interpolation="linear")
        NP.at_time(0.61)                                    # a new view is built on the device too
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for line in (False, True):
        _equal(first[line], again[line], f"repeat line={line}")
    _equal(uni, uni2, "repeat uniform")


def test_at_time_view_rows():
    from nersemble_b200 import ops
    P = oracle_params(KNOBS)
    NP = native_from_oracle(P, DEV)
    T = NP.n_timesteps
    for k in range(T):
        V = NP.at_time(k / (T - 1))
        assert V.n_timesteps == 1 and V.tables is NP.tables and V.field_packed is NP.field_packed
        assert torch.equal(V.blend_codes[0], NP.blend_codes[k]) and torch.equal(V.deform_code_bias[0], NP.deform_code_bias[k])
        assert torch.equal(V.warp_codes[0], NP.warp_codes[k])
    V = NP.at_time(0.5)
    assert V is NP.at_time(0.5)                             # cached
    i0, i1, lam = ops.time_lerp(0.5, T)
    assert torch.equal(V.blend_codes[0], ops._lerp_f32(NP.blend_codes[i0], NP.blend_codes[i1], lam))
    NP.blend_codes.mul_(1.0)                                # a new parameter version rebuilds the view
    assert NP.at_time(0.5) is not V


def _model(deform):
    from test_gpu_flow import _cache_and_model
    return _cache_and_model(deform)


@pytest.mark.parametrize("deform", [True, False])
def test_model_time_interpolation(deform):
    from nersemble_b200 import ops
    m, cache, sampler, (H, W) = _model(deform)
    assert m.time_interpolation == "nearest"
    bundle, _ = sampler.camera_ray_bundle(3)                    # camera 1, timestep 1: an integer time
    # without a deformation field, mixed linear times take get_outputs' general path (sampler + per-sample codes): its
    # nearest counterpart is the general path too
    m.use_fused_render = deform
    near = m.get_outputs_for_camera_ray_bundle(bundle)
    m.use_fused_render = True
    m.time_interpolation = "linear"
    lin = m.get_outputs_for_camera_ray_bundle(bundle)
    for k in ("rgb", "accumulation", "depth", "deformation"):
        if k in lin:
            assert torch.equal(near[k], lin[k]), k
    # a fractional frame: the mixed-time kernels and the at_time view agree, and the view is what ops renders
    t = 0.4
    bundle.times = torch.full_like(bundle.times, t)
    frac = m.get_outputs_for_camera_ray_bundle(bundle)
    assert (frac["rgb"] - lin["rgb"]).abs().max() > 0
    m.frame_table_min_rays = 0                                  # the whole frame on the at_time view
    frame = m.get_outputs_for_camera_ray_bundle(bundle)
    if deform:
        assert (frac["rgb"] - frame["rgb"]).norm(dim=-1).max() < RGB_L2
    rb = bundle.get_row_major_sliced_ray_bundle(0, H * W)
    near_p, far_p = m.sampler.eval_planes(rb, m.config.near_plane, m.config.far_plane)
    og = m.occupancy_grid
    wh, wd = m._windows()
    want = ops.render_rays(m.native_params(), rb.origins.reshape(-1, 3), rb.directions.reshape(-1, 3), m._ray_times(rb),
                           window_hash=wh, window_deform=wd, use_deformation=deform, sampler="occupancy",
                           near_planes=near_p, far_planes=far_p, binaries=og.binaries, aabbs=og.aabbs,
                           step=m.config.render_step_size, cone_angle=m.config.cone_angle, uniform_time=t,
                           time_interpolation="linear", **m._blend_opts())
    assert torch.equal(frame["rgb"].reshape(-1, 3), want["rgb"])
    # training and flow
    m.frame_table_min_rays = 16384
    with pytest.raises(NotImplementedError, match="linear"):
        m.render_flow(bundle, 2)
    m.train()
    m.sampler.train()
    with pytest.raises(ValueError, match="time_interpolation"):
        m.get_outputs(bundle.get_row_major_sliced_ray_bundle(0, 64))
