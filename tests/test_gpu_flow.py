"""Scene flow and optical flow of a render (ops.render_flow: nsb_flow_select -> nsb_deform_inverse -> nsb_flow_composite) on
the GPU: the selection against the oracle on a fixed-stride and an occupancy render, the compositing against the float64
oracle on the kernel's own inverse outputs, a rigid rotation between two timesteps with a known answer, flow to the
rays' own timestep, random heads, repeatability, no host synchronisation, unchanged render outputs, and the model method."""
import math

import pytest
import torch

from conftest import native_from_oracle, oracle_params
from deform_inverse_oracle import rigid_params
from flow_oracle import composite, project, ray_directions, select
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = dict(seed=19980801, n_timesteps=24, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
             deform_last_scale=2e-2)      # the random heads of test_gpu_deform_inverse.py
WH, WD = 32.0, 7.0
MW = 1e-3


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@pytest.fixture(scope="module")
def deformed():
    P = oracle_params(KNOBS)
    return P, native_from_oracle(P, DEV)


def _rays(R, seed):
    from oracle.gen_golden import ring_rays
    o, d, t, _ = ring_rays(R, seed)
    return o.to(DEV), d.to(DEV), t.reshape(-1).to(DEV)


def _fixed(NP, o, d, t, **kw):
    from nersemble_b200 import ops
    return ops.render_rays(NP, o, d, t, window_hash=WH, window_deform=WD, sampler="fixed", n_per_ray=64, near_plane=0.2,
                           step=0.08, **kw)


def _occupancy(P, NP, o, d, t):
    from nersemble_b200 import ops
    from oracle.gen_golden import blob_grid
    R = o.shape[0]
    near = torch.full((R,), 0.2, device=DEV); far = torch.full((R,), 1e3, device=DEV)
    return ops.render_rays(NP, o, d, t, window_hash=WH, window_deform=WD, sampler="occupancy", near_planes=near,
                           far_planes=far, binaries=blob_grid(7)[None].to(DEV), aabbs=P.aabb.reshape(1, 6).to(DEV), step=0.011)


def _camera(center, dist, fx, H, W, azimuth=0.6):
    """A pinhole looking at `center` from `dist` away (-z forward, +y up): (intrinsics, camera_to_world [3,4]) float64."""
    c = torch.as_tensor(center, dtype=torch.float64)
    eye = c + dist * torch.tensor([math.sin(azimuth), 0.25, math.cos(azimuth)], dtype=torch.float64)
    fwd = (c - eye) / (c - eye).norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64)); right = right / right.norm()
    up = torch.linalg.cross(right, fwd)
    return (fx, fx * 1.02, W / 2 + 0.3, H / 2 - 0.2), torch.cat([torch.stack([right, up, -fwd], -1), eye[:, None]], -1)


def _camera_rays(cam, H, W):
    rows, cols = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    d = ray_directions(cam[0], cam[1], rows.reshape(-1), cols.reshape(-1)).float()
    o = cam[1][:, 3].float().expand(H * W, 3).contiguous()
    return o.to(DEV), d.to(DEV)


def _packed_view(res):
    """The render's per-sample arrays over their full capacity and the device sample count (read here: tests may sync)."""
    b = res["_buffers"]
    return b, int(b["header"][2])


def _check_selection(res, flow, o, d):
    b, n_total = _packed_view(res)
    want = select(res["packed_info"], b["t_starts"], b["t_ends"], b["weights"], b["offsets"], o, d, n_total, MW)
    n = want["n_selected"]
    print(f"selection: {n} of {n_total} samples (capacity {b['capacity']})")
    assert 0 < n < n_total
    assert int(flow["_n_selected"]) == n
    assert torch.equal(flow["_ray_sel"].cpu(), want["ray_sel"])
    assert torch.equal(flow["_sel_index"][:n].cpu(), want["sel_index"])
    assert torch.equal(flow["_init"][:n].cpu(), want["init"]) and torch.equal(flow["_targets"][:n].cpu(), want["targets"])


def test_selection_matches_the_oracle_fixed_stride(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = _rays(600, 3)
    res = _fixed(NP, o, d, t)
    flow = ops.render_flow(NP, res, o, d, t, time_to=0.4, window_deform=WD)
    _check_selection(res, flow, o, d)


def test_selection_matches_the_oracle_occupancy_and_ignores_slots_past_n_total(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = _rays(900, 4)
    res = _occupancy(P, NP, o, d, t)
    b, n_total = _packed_view(res)
    assert n_total < b["capacity"]
    for k in ("t_starts", "t_ends", "weights", "offsets"):
        b[k][n_total:] = float("nan")
    b["weights"][n_total:] = 1.0          # would be selected if read
    flow = ops.render_flow(NP, res, o, d, t, time_to=0.4, window_deform=WD)
    _check_selection(res, flow, o, d)


def _oracle_of(res, flow, camera=None):
    inv = flow["_inverse"]
    return composite(flow["_ray_sel"], flow["_sel_index"], flow["_init"], inv["positions"], inv["status"],
                     res["_buffers"]["weights"], camera)


def _close(got, want, what, rtol=1e-5):
    got = got.cpu().double().reshape(want.shape)
    atol = rtol * max(want.abs().max().item(), 1e-30)
    err = (got - want).abs().max().item()
    print(f"{what}: max |got - oracle| {err:.3e} (scale {want.abs().max().item():.3e})")
    torch.testing.assert_close(got, want, rtol=rtol, atol=atol)


def test_compositing_matches_the_oracle(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = _rays(600, 5)
    cam = _camera((0.0, 0.0, 0.0), 9.0, 700.0, 64, 64)
    res = _fixed(NP, o, d, t)
    flow = ops.render_flow(NP, res, o, d, t, time_to=0.8, window_deform=WD, camera=cam)
    want = _oracle_of(res, flow, cam)
    assert (want["flow_weight"] > 0).float().mean() > 0.3
    for k in ("scene_flow", "flow_weight", "optical_flow"):
        _close(flow[k], want[k], k)


def _rotation(r):
    th = (r * r).sum().clamp_min(1e-4).sqrt()
    K = torch.tensor([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    return torch.eye(3) + (th.sin() / th) * K + ((1 - th.cos()) / th ** 2) * (K @ K)


def _two_frame_params():
    """The fixture of test_gpu_deform_inverse.py: timestep 0 the identity, timestep 1 a rotation R about the box origin
    (unit-cube box), one geometry, a smooth field (levels of resolution <= 33)."""
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


def test_rigid_rotation_between_two_timesteps():
    from nersemble_b200 import ops
    P, Rm = _two_frame_params()
    NP = native_from_oracle(P, DEV)
    H, W = 40, 48
    cam = _camera((0.5, 0.5, 0.5), 3.0, 60.0, H, W)
    o, d = _camera_rays(cam, H, W)
    t = torch.zeros(H * W, device=DEV)
    res = ops.render_rays(NP, o, d, t, window_hash=WH, window_deform=WD, sampler="fixed", n_per_ray=96, near_plane=0.0,
                          step=0.02)
    flow = ops.render_flow(NP, res, o, d, t, time_to=1.0, window_deform=WD, camera=cam)
    n = int(flow["_n_selected"])
    inv = flow["_inverse"]
    assert n > 1000 and bool(inv["converged"][:n].all())
    x = flow["_init"][:n].cpu().double()
    w = res["_buffers"]["weights"].cpu().double()[flow["_sel_index"][:n].cpu()]
    y = x @ Rm.double()                                                   # rows: R^T x
    ray = torch.repeat_interleave(torch.arange(H * W), flow["_ray_sel"][:, 1].cpu())
    Wr = torch.zeros(H * W, dtype=torch.float64).index_add_(0, ray, w)
    has = Wr > 0
    sf = torch.zeros((H * W, 3), dtype=torch.float64).index_add_(0, ray, w[:, None] * (y - x))
    err = (flow["scene_flow"].cpu().double()[has] - sf[has] / Wr[has, None]).abs().max().item()
    p0, f0 = project(x, *cam)
    p1, f1 = project(y, *cam)
    assert f0.all() and f1.all()
    of = torch.zeros((H * W, 2), dtype=torch.float64).index_add_(0, ray, w[:, None] * (p1 - p0))
    oerr = (flow["optical_flow"].cpu().double()[has] - of[has] / Wr[has, None]).abs().max().item()
    print(f"rigid rotation: {int(has.sum())} rays with flow, {n} samples; scene flow error {err:.3e}, optical flow error "
          f"{oerr:.3e} px (flow up to {(of[has] / Wr[has, None]).abs().max().item():.2f} px)")
    assert err <= 1e-5 and oerr <= 1e-3
    # flow_weight: the weight of the samples at or above min_weight
    b, n_total = _packed_view(res)
    wa = b["weights"][:n_total].cpu().double()
    ri = b["ray_indices"][:n_total].cpu().long()
    want_w = torch.zeros(H * W, dtype=torch.float64).index_add_(0, ri, torch.where(wa >= MW, wa, torch.zeros_like(wa)))
    torch.testing.assert_close(flow["flow_weight"].cpu().double()[:, 0], want_w, rtol=1e-5, atol=1e-6)
    assert (flow["scene_flow"][~has.to(DEV)] == 0).all() and (flow["optical_flow"][~has.to(DEV)] == 0).all()


def test_flow_to_the_rays_own_timestep(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, _ = _rays(800, 6)
    t0 = 5.0 / 23.0
    t = torch.full((800,), t0, device=DEV)
    res = _fixed(NP, o, d, t)
    tol = 1e-4
    flow = ops.render_flow(NP, res, o, d, t, time_to=t0, window_deform=WD, tol=tol)
    n = int(flow["_n_selected"])
    inv = flow["_inverse"]
    it = inv["iterations"][:n]
    assert n > 1000 and bool(inv["converged"][:n].all())
    moved = (inv["positions"][:n] - flow["_init"][:n]).abs().amax(-1)
    assert (moved[it == 0] == 0).all()
    ray = torch.repeat_interleave(torch.arange(800, device=DEV), flow["_ray_sel"][:, 1])
    any_iter = torch.zeros(800, dtype=torch.int64, device=DEV).index_add_(0, ray, (it > 0).long()) > 0
    ext = max(NP.aabb_list[3 + k] - NP.aabb_list[k] for k in range(3))
    sf = flow["scene_flow"].abs().amax(-1)
    print(f"own timestep: {int((it > 0).sum())} of {n} samples needed an iteration (wgmma render offsets vs mma.sync "
          f"inverse offsets); max |x' - x| {moved.max().item():.3e}, max |scene_flow| {sf.max().item():.3e} "
          f"(tol x extent {tol * ext:.3e})")
    assert (sf[~any_iter] == 0).all()
    # a sample needs an iteration when the two roles' offsets differ by about tol x extent, and Newton then moves it by
    # about that difference
    assert (sf[any_iter] < 2 * tol * ext).all()


def test_random_heads_converge_and_match_the_oracle(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = _rays(1000, 7)
    res = _fixed(NP, o, d, t)
    cam = _camera((0.0, 0.0, 0.0), 9.0, 700.0, 64, 64, azimuth=1.3)
    flow = ops.render_flow(NP, res, o, d, t, time_to=0.9, window_deform=WD, camera=cam)
    n = int(flow["_n_selected"])
    w = res["_buffers"]["weights"][flow["_sel_index"][:n]]
    conv = flow["_inverse"]["converged"][:n]
    frac = (w * conv).sum().item() / w.sum().item()
    print(f"random heads: {n} selected, {conv.float().mean().item():.5f} of them and {frac:.5f} of their weight converged, "
          f"status {torch.bincount(flow['_inverse']['status'][:n].long()).tolist()}")
    assert frac >= 0.99
    want = _oracle_of(res, flow, cam)
    for k in ("scene_flow", "flow_weight", "optical_flow"):
        _close(flow[k], want[k], f"random heads {k}")


def test_repeatable_sync_free_and_render_outputs_unchanged(deformed):
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = _rays(500, 8)
    cam = _camera((0.0, 0.0, 0.0), 9.0, 700.0, 64, 64)
    plain = _fixed(NP, o, d, t)
    res = _fixed(NP, o, d, t)
    first = ops.render_flow(NP, res, o, d, t, time_to=0.3, window_deform=WD, camera=cam)
    second = ops.render_flow(NP, res, o, d, t, time_to=0.3, window_deform=WD, camera=cam)
    for k in ("scene_flow", "flow_weight", "optical_flow", "_ray_sel", "_n_selected"):
        assert torch.equal(first[k], second[k]), k
    n = int(first["_n_selected"])
    for k in ("_sel_index", "_targets", "_init"):
        assert torch.equal(first[k][:n], second[k][:n]), k
    for k in ("positions", "residual", "iterations", "status"):
        assert torch.equal(first["_inverse"][k][:n], second["_inverse"][k][:n]), k
    for k in ("rgb", "depth", "accumulation", "deformation"):
        assert torch.equal(res[k], plain[k]), k
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r2 = _fixed(NP, o, d, t)
        f2 = ops.render_flow(NP, r2, o, d, t, time_to=0.3, window_deform=WD, camera=cam)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(f2["scene_flow"], first["scene_flow"]) and torch.equal(f2["optical_flow"], first["optical_flow"])


def _cache_and_model(deform):
    from nersemble_b200.plugin import DeviceImageCache, DeviceRaySampler
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P = oracle_params(dict(KNOBS, n_timesteps=4))
    m = make_model(T=4, log2T=14, eval_num_rays_per_chunk=500)
    load_oracle_params_into(m, P)
    m.config.use_deformation_field = deform
    m = m.to(DEV).eval()
    occ = blob_grid(5)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(DEV))
    H, W, T = 24, 32, 4
    cams = [_camera((0.0, 0.0, 0.0), 9.0, 150.0, H, W, azimuth=a) for a in (0.3, 2.0)]
    intr = torch.tensor([c[0] for c in cams]); c2w = torch.stack([c[1] for c in cams]).float()
    n_img = 2 * T
    cache = DeviceImageCache(torch.zeros((n_img, H, W, 3), dtype=torch.uint8), torch.arange(n_img) % 2,
                             (torch.arange(n_img) // 2).float() / (T - 1), intr, c2w, device=DEV)
    return m, cache, DeviceRaySampler(cache), (H, W)


@pytest.mark.parametrize("deform", [True, False])
def test_model_render_flow(deform):
    m, cache, sampler, (H, W) = _cache_and_model(deform)
    bundle, _ = sampler.camera_ray_bundle(3)                    # camera 1, timestep 1
    img = m.get_outputs_for_camera_ray_bundle(bundle)
    out = m.render_flow(bundle, 2, intrinsics=cache.intrinsics[1], camera_to_world=cache.camera_to_world[1])
    assert out["scene_flow"].shape == (H, W, 3) and out["flow_weight"].shape == (H, W, 1)
    assert out["optical_flow"].shape == (H, W, 2)
    assert set(out) == set(img) | {"scene_flow", "flow_weight", "optical_flow"}
    for k in img:
        assert torch.equal(out[k], img[k]), k
    assert (img["accumulation"] > 0).float().mean() > 0.05
    if deform:
        assert torch.isfinite(out["scene_flow"]).all() and torch.isfinite(out["optical_flow"]).all()
        assert (out["flow_weight"] <= out["accumulation"] + 1e-6).all()
        assert out["scene_flow"].abs().max() > 0
        plain = m.render_flow(bundle, 2)
        assert "optical_flow" not in plain and torch.equal(plain["scene_flow"], out["scene_flow"])
    else:
        assert (out["scene_flow"] == 0).all() and (out["optical_flow"] == 0).all()
        assert torch.equal(out["flow_weight"], out["accumulation"])
    with pytest.raises(ValueError, match="timestep"):
        m.render_flow(bundle, 4)
