"""The deformation's input gradient (nsb_deform_input_grad) and observation-space normals on the GPU: a rigid warp with a
known answer, J^T u and the normals against the CPU oracle (autograd through oracle.pipeline, kernel precision), tile
edges, and the guarantees that nothing else moved (canonical outputs bit-identical, no host synchronisation).

The reference initialises the deformation heads with U(+-1e-5): J is ~0 on fresh parameters and a test on them proves
nothing.  The parameters here draw the heads from U(+-2e-2) (offsets of a few percent of the box), and the tests assert that
the oracle's |J| is at least 0.1 on most samples."""
import pytest
import torch

from conftest import native_from_oracle, oracle_params
from deform_jacobian_oracle import jacobian_norm, observation_normals, offsets_vjp
from normals_oracle import composite_normals
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = dict(seed=19980801, n_timesteps=24, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
             deform_last_scale=2e-2)      # the default box is the non-cubic one (4.7 x 3.6 x 4.5): a misplaced D^-1 fails


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
    return o, d, t


def _angles(a, b):
    return torch.rad2deg(torch.acos((a * b).sum(-1).clamp(-1.0, 1.0)))


def _check_angles(got, want, g_ref, what):
    """The bars of the canonical normals tests: at least 99.9 % within 1 degree and all within 5 degrees, over samples
    whose oracle gradient norm is at least 1e-3 of the median."""
    gn = g_ref.norm(dim=-1)
    keep = gn >= 1e-3 * gn[gn > 0].median()
    ang = _angles(got[keep], want[keep])
    frac = (ang <= 1.0).float().mean().item()
    assert frac >= 0.999 and ang.max().item() <= 5.0, (what, frac, ang.max().item(), int(keep.sum()))


def _rotation(r: torch.Tensor) -> torch.Tensor:
    """The matrix the SE(3) map applies to p: I + f1 K + f2 K^2 with theta^2 clamped at 1e-4 (util/pytorch3d.py)."""
    th = (r * r).sum().clamp_min(1e-4).sqrt()
    K = torch.tensor([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    return torch.eye(3) + (th.sin() / th) * K + ((1 - th.cos()) / th ** 2) * (K @ K)


def _rigid_params(r, v):
    """Unit-cube box, stem weights and biases zero (a5 = 0), head biases (r, v): the warp is x = R p_n + V v everywhere."""
    P = pl.random_params(n_timesteps=2, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
                         aabb=((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)))
    for w, b in zip(P.deform_w, P.deform_b):
        w.zero_(); b.zero_()
    P.r_b.copy_(torch.tensor(r)); P.v_b.copy_(torch.tensor(v))
    return P


@pytest.mark.parametrize("r", [(0.1, -0.15, 0.12), (3e-3, -2e-3, 1e-3)], ids=["rotation", "clamped_theta"])
def test_rigid_warp_rotates_the_normals(r):
    """x = R p_n + t, so n_obs = R^T n_canonical for every sample whose warped position is inside the box, to 1e-4 per
    component; the second case has theta^2 < 1e-4 (the clamp branch of the exponential map)."""
    from nersemble_b200 import ops
    P = _rigid_params(r, (0.02, -0.03, 0.01))
    NP = native_from_oracle(P, DEV)
    gen = torch.Generator().manual_seed(3)
    n = 2000
    pos = (0.35 + 0.3 * torch.rand((n, 3), generator=gen)).to(DEV)
    times = torch.rand((n,), generator=gen).to(DEV)
    kw = dict(window_hash=32.0, positions=pos, sample_times=times)
    off = ops.field_forward(NP, window_deform=7.0, want=("offsets",), **kw)["offsets"]
    xw = pos + off
    assert ((xw > 0) & (xw < 1)).all()
    can = ops.field_normals(NP, offsets=off, **kw)["normals"]
    obs = ops.field_normals(NP, offsets=off, space="observation", window_deform=7.0, **kw)["normals"]
    R = _rotation(torch.tensor(r)).to(DEV)
    want = can @ R            # rows: R^T n
    want = want / want.norm(dim=-1, keepdim=True)
    assert (obs - want).abs().max().item() <= 1e-4, (obs - want).abs().max().item()
    assert (obs - can).abs().max().item() > 10 * 1e-4 or max(abs(c) for c in r) < 1e-2


def _vjp_errors(got, want):
    rel = (got - want).norm(dim=-1) / want.norm(dim=-1).clamp_min(1e-20)
    return rel, (rel > 2e-2).sum().item()


@pytest.mark.parametrize("window", [None, 3.5])
def test_vjp_matches_the_oracle_table_codes(deformed, window):
    """Ray-based samples, T = 24 timesteps mixed per ray.  A stem ReLU that flips under the fp16 rounding of the
    recomputed activations moves a few rows: 99 % within 2e-2 relative L2, all within 2e-1."""
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = _rays(64, 3)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 40, 0.1, near=0.2)
    n = ts.shape[0]
    pos = o[ri] + d[ri] * (ts + te)[:, None] * 0.5
    wc = P.time_emb_deform[pl.timesteps_from_times(t[ri], P.n_timesteps)]
    u = torch.randn((n, 3), generator=torch.Generator().manual_seed(1))
    jn = jacobian_norm(P, pos, wc, window)
    assert (jn >= 0.1).float().mean() > 0.9, jn.median()
    want = offsets_vjp(P, pos, wc, window, u)
    got = ops.deform_input_grad(NP, u.to(DEV), window_deform=window, origins=o.to(DEV), directions=d.to(DEV),
                                ray_times=t.to(DEV), t_starts=ts.to(DEV), t_ends=te.to(DEV), ray_indices=ri.to(DEV)).cpu()
    rel, n_off = _vjp_errors(got, want)
    print(f"J^T u, table codes, window {window}: {n_off} of {n} rows above 2e-2, worst {rel.max().item():.3e}")
    assert n_off <= 0.01 * n and rel.max().item() <= 2e-1, (n_off, n, rel.max().item())


@pytest.mark.parametrize("window", [None, 3.5])
def test_vjp_matches_the_oracle_per_sample_codes(deformed, window):
    from nersemble_b200 import ops
    P, NP = deformed
    gen = torch.Generator().manual_seed(7)
    n = 3000
    pos = P.aabb[0] + (torch.rand((n, 3), generator=gen) * 1.1 - 0.05) * (P.aabb[1] - P.aabb[0])
    wc = torch.randn((n, 128), generator=gen) * 0.1
    u = torch.randn((n, 3), generator=gen)
    assert (jacobian_norm(P, pos, wc, window) >= 0.1).float().mean() > 0.9
    want = offsets_vjp(P, pos, wc.half().float(), window, u)
    got = ops.deform_input_grad(NP, u.to(DEV), window_deform=window, positions=pos.to(DEV), sample_warp_codes=wc.to(DEV)).cpu()
    rel, n_off = _vjp_errors(got, want)
    print(f"J^T u, per-sample codes, window {window}: {n_off} of {n} rows above 2e-2, worst {rel.max().item():.3e}")
    assert n_off <= 0.01 * n and rel.max().item() <= 2e-1, (n_off, n, rel.max().item())


def test_vjp_tile_edges_and_device_count(deformed):
    """n = 1, 127, 129 give the rows of the large call (a row's result does not depend on its tile), and with a device
    sample count below the buffer size the rows beyond it keep what they held."""
    from nersemble_b200 import ops
    P, NP = deformed
    gen = torch.Generator().manual_seed(9)
    n = 300
    pos = (P.aabb[0] + torch.rand((n, 3), generator=gen) * (P.aabb[1] - P.aabb[0])).to(DEV)
    times = torch.rand((n,), generator=gen).to(DEV)
    u = torch.randn((n, 3), generator=gen).to(DEV)
    full = ops.deform_input_grad(NP, u, window_deform=7.0, positions=pos, sample_times=times)
    assert torch.isfinite(full).all()
    for k in (1, 127, 129):
        part = ops.deform_input_grad(NP, u[:k], window_deform=7.0, positions=pos[:k], sample_times=times[:k])
        assert torch.equal(part, full[:k]), k
    out = torch.full((n, 3), -77.0, device=DEV)
    count = torch.tensor([200], dtype=torch.int64, device=DEV)
    ops.deform_input_grad(NP, u, window_deform=7.0, positions=pos, sample_times=times, n_samples_dev=count, out=out)
    assert torch.equal(out[:200], full[:200]) and (out[200:] == -77.0).all()
    assert torch.equal(full, ops.deform_input_grad(NP, u, window_deform=7.0, positions=pos, sample_times=times))


def test_field_api_observation_normals_match_the_oracle(deformed):
    """Explicit positions, table codes (timestep stack), normalised space; a band of positions around the box so that
    some warped positions leave it: those give exactly zero."""
    from nersemble_b200 import ops
    P, NP = deformed
    gen = torch.Generator().manual_seed(11)
    n = 3000
    pos = P.aabb[0] + (torch.rand((n, 3), generator=gen) * 1.06 - 0.03) * (P.aabb[1] - P.aabb[0])
    times = torch.rand((n,), generator=gen)
    tsi = pl.timesteps_from_times(times, P.n_timesteps)
    kw = dict(window_hash=32.0, positions=pos.to(DEV), sample_times=times.to(DEV))
    off = ops.field_forward(NP, window_deform=7.0, want=("offsets",), **kw)["offsets"]
    got = ops.field_normals(NP, offsets=off, space="observation", window_deform=7.0, **kw)["normals"].cpu()
    want, g, sel = observation_normals(P, pos, P.time_emb_deform[tsi], P.time_emb[tsi], 32.0, 7.0, offsets=off.cpu())
    assert 20 < (~sel).sum() < n // 2
    assert (got[~sel] == 0).all()
    _check_angles(got[sel], want[sel], g[sel], "field API, observation space")


def _render(NP, o, d, t, **kw):
    from nersemble_b200 import ops
    return ops.render_rays(NP, o.to(DEV), d.to(DEV), t.to(DEV), window_hash=32.0, window_deform=7.0, sampler="fixed",
                           n_per_ray=48, near_plane=0.2, step=0.1, want_normals=True, **kw)


@pytest.mark.parametrize("mode", ["stack", "line", "uniform"])
def test_rendered_observation_normals_match_the_oracle(deformed, mode):
    """World-space per-sample normals of render samples and their composite, through the timestep stack, the line gather
    (fp16 member weights in the oracle too) and the frame table of a uniform time."""
    P, NP = deformed
    R = 96
    o, d, t = _rays(R, 3)
    kw = {}
    if mode == "uniform":
        t = torch.full((R, 1), 5.0 / 23.0)
        kw["uniform_time"] = 5.0 / 23.0
    res = _render(NP, o, d, t, normals_space="observation", line_gather=mode == "line", **kw)
    pk = res.packed()
    ri = pk["ray_indices"].cpu().long()
    pos = o[ri] + d[ri] * (pk["t_starts"] + pk["t_ends"]).cpu()[:, None] * 0.5
    tsi = pl.timesteps_from_times(t[ri], P.n_timesteps)
    want, g, sel = observation_normals(P, pos, P.time_emb_deform[tsi], P.time_emb[tsi], 32.0, 7.0, world_space=True,
                                       blend_fp16=mode == "line", offsets=pk["offsets"].cpu())
    got = pk["normals"].cpu()
    assert (~sel).sum() > 100 and (got[~sel] == 0).all()
    _check_angles(got[sel], want[sel], g[sel], mode)
    own = composite_normals(got, pk["weights"].cpu(), ri, R)
    assert (res["normals"].cpu() - own).norm(dim=-1).max() <= 1e-5
    ref = composite_normals(want, pk["weights"].cpu(), ri, R)
    hit = res["accumulation"].cpu()[:, 0] >= 0.5
    if hit.any():
        assert ((res["normals"].cpu() - ref)[hit].norm(dim=-1) > 1e-2).float().mean() <= 0.02


def test_nothing_else_moved(deformed):
    """Canonical is the default and the same bits as before; without deformation both spaces are the same bits;
    observation renders repeat bit for bit, leave rgb / depth / accumulation alone and issue no host synchronisation."""
    from nersemble_b200 import ops
    P, NP = deformed
    o, d, t = (v.to(DEV) for v in _rays(256, 4))
    kw = dict(window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=64, near_plane=0.2, step=0.02, want_normals=True)
    plain = ops.render_rays(NP, o, d, t, **kw)
    can = ops.render_rays(NP, o, d, t, normals_space="canonical", **kw)
    obs = ops.render_rays(NP, o, d, t, normals_space="observation", **kw)       # warm-up: packs the posenc block
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        obs2 = ops.render_rays(NP, o, d, t, normals_space="observation", **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(plain["normals"], can["normals"])
    assert torch.equal(obs["normals"], obs2["normals"]) and not torch.equal(obs["normals"], can["normals"])
    assert torch.equal(obs.packed()["normals"], obs2.packed()["normals"])
    for k in ("rgb", "accumulation", "depth", "deformation", "num_samples_per_ray"):
        assert torch.equal(obs[k], plain[k]), k
    nd_c = ops.render_rays(NP, o, d, t, use_deformation=False, **kw)
    nd_o = ops.render_rays(NP, o, d, t, use_deformation=False, normals_space="observation", **kw)
    assert torch.equal(nd_c["normals"], nd_o["normals"]) and torch.equal(nd_c.packed()["normals"], nd_o.packed()["normals"])
    # field API
    pk = plain.packed()
    skw = dict(window_hash=32.0, origins=o, directions=d, ray_times=t, t_starts=pk["t_starts"], t_ends=pk["t_ends"],
               ray_indices=pk["ray_indices"])
    a = ops.field_normals(NP, offsets=pk["offsets"], **skw)["normals"]
    b = ops.field_normals(NP, offsets=pk["offsets"], space="canonical", window_deform=7.0, **skw)["normals"]
    c = ops.field_normals(NP, space="observation", **skw)["normals"]           # no offsets: no deformation
    assert torch.equal(a, b) and torch.equal(c, ops.field_normals(NP, **skw)["normals"])


def test_model_render_normals_space():
    """NeRSembleNGPModel.render_normals_space through get_outputs (fused eval, packed eval, training forward) and
    get_outputs_for_camera_ray_bundle: observation differs from canonical, the other outputs do not change, and the
    two eval paths agree on rays that hit the surface.  The training forward keeps other samples (its visibility
    pre-pass) and gathers table lines: there the observation channel has to agree with the fused one as well as the
    canonical channel does."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P = oracle_params(dict(KNOBS, n_timesteps=4))
    m = make_model(T=4, log2T=14, eval_num_rays_per_chunk=500)
    load_oracle_params_into(m, P)
    m = m.to(DEV).eval()
    occ = blob_grid(5)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(DEV))
    R = 300
    o, d, t = _rays(R, 8)
    rb = RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV),
                   camera_indices=torch.zeros(R, 1, dtype=torch.long, device=DEV), times=t.to(DEV))
    m.render_normals = True
    assert m.render_normals_space == "canonical"
    got = {}
    can_of = {}
    for fused in (True, False):
        m.use_fused_render = fused
        with torch.no_grad():
            m.render_normals_space = "canonical"
            can = can_of[fused] = m.get_outputs(rb)
            m.render_normals_space = "observation"
            obs = got[fused] = m.get_outputs(rb)
        assert set(can) == set(obs) and torch.isfinite(obs["normals"]).all()
        assert not torch.equal(can["normals"], obs["normals"])
        for k in ("rgb", "accumulation", "depth", "deformation"):
            assert torch.equal(can[k], obs[k]), (fused, k)
    m.train(); m.sampler.eval()
    got["train"] = m.get_outputs(rb)
    m.render_normals_space = "canonical"
    can_of["train"] = m.get_outputs(rb)
    m.render_normals_space = "observation"
    assert got["train"]["normals"].grad_fn is None and got["train"]["rgb"].grad_fn is not None
    m.eval()
    hit = got[True]["accumulation"][:, 0] >= 0.5
    assert hit.sum() > 50
    err = (got[True]["normals"] - got[False]["normals"])[hit].norm(dim=-1)
    assert (err > 2e-2).float().mean().item() <= 0.02, (err.max().item(), int(hit.sum()))
    err_obs = (got[True]["normals"] - got["train"]["normals"])[hit].norm(dim=-1)
    err_can = (can_of[True]["normals"] - can_of["train"]["normals"])[hit].norm(dim=-1)
    print(f"train vs fused, rays hit {int(hit.sum())}: observation mean {err_obs.mean().item():.3e}, canonical mean {err_can.mean().item():.3e}")
    assert err_obs.mean().item() <= 2.0 * err_can.mean().item() + 1e-3, (err_obs.mean().item(), err_can.mean().item())
    m.use_fused_render = True
    H, W = 20, 30
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1.5, 1.5, W), indexing="ij")
    cam_o = torch.tensor([0.0, 0.0, 9.0]).expand(H, W, 3).contiguous()
    cam_d = torch.stack([xs, ys, torch.full_like(xs, -9.0)], -1); cam_d = cam_d / cam_d.norm(dim=-1, keepdim=True)
    cam = RayBundle(origins=cam_o.to(DEV), directions=cam_d.to(DEV), pixel_area=torch.ones(H, W, 1, device=DEV),
                    camera_indices=torch.zeros(H, W, 1, dtype=torch.long, device=DEV), times=torch.full((H, W, 1), 0.34, device=DEV))
    img_obs = m.get_outputs_for_camera_ray_bundle(cam)
    m.render_normals_space = "canonical"
    img_can = m.get_outputs_for_camera_ray_bundle(cam)
    assert img_obs["normals"].shape == (H, W, 3) and not torch.equal(img_obs["normals"], img_can["normals"])
    for k in img_can:
        if k != "normals":
            assert torch.equal(img_obs[k], img_can[k]), k


def test_rotation_between_two_timesteps_turns_the_observation_normals():
    """Two timesteps whose deformations differ by a pure rotation (timestep 0: identity; timestep 1: R about the box
    origin; unit-cube box).  Frame 1 observes the points p1 = R^T p0, which warp to the canonical points frame 0 sees:
    the canonical normals of the two frames are the same, the observation normals differ by exactly that rotation --
    per sample and in the composited channel."""
    from nersemble_b200 import ops
    r = torch.tensor([0.0625, -0.125, 0.25])        # exact in fp16, the heads' operand type
    P = _rigid_params((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    # unit 0 of every stem layer carries code[0] to the heads: a5[0] = code_t[0], r = r_vec * a5[0]
    P.deform_w[0][0, 45] = 1.0
    for l in (1, 2, 3, 5):
        P.deform_w[l][0, 0] = 1.0
    P.deform_w[4][0, 173] = 1.0
    P.r_w.zero_(); P.v_w.zero_(); P.r_w[:, 0] = r
    P.time_emb_deform.zero_(); P.time_emb_deform[1, 0] = 1.0
    P.time_emb[1] = P.time_emb[0]                   # one geometry: the frames only differ by the warp
    NP = native_from_oracle(P, DEV)
    Rm = _rotation(r)
    gen = torch.Generator().manual_seed(13)
    n_rays, per = 40, 25
    n = n_rays * per
    p0 = 0.35 + 0.3 * torch.rand((n, 3), generator=gen)
    p1 = p0 @ Rm                                    # rows: R^T p0
    assert ((p1 > 0.02) & (p1 < 0.98)).all()
    info = torch.stack([torch.arange(n_rays) * per, torch.full((n_rays,), per)], -1).to(DEV)
    w = torch.rand((n,), generator=gen).to(DEV)
    res = {}
    for frame, pos in ((0, p0), (1, p1)):
        kw = dict(window_hash=32.0, positions=pos.to(DEV), sample_times=torch.full((n,), float(frame), device=DEV))
        off = ops.field_forward(NP, window_deform=7.0, want=("offsets",), **kw)["offsets"]
        x = pos.to(DEV) + off
        res[frame] = {"x": x}
        for space in ("canonical", "observation"):
            res[frame][space] = ops.field_normals(NP, offsets=off, space=space, window_deform=7.0, packed_info=info,
                                                  weights=w, **kw)
    assert (res[0]["x"] - res[1]["x"]).abs().max() < 2e-6       # the same canonical points
    Rd = Rm.to(DEV)

    def close(a, b, tol, frac):
        """The two frames' hash inputs differ in the last bits, so a few samples sit in different cells of a fine level
        and their gradients differ: `frac` of the rows within `tol`."""
        return ((a - b).abs().amax(-1) <= tol).float().mean().item() >= frac

    for key, tol, frac in (("normals", 2e-3, 0.95), ("ray_normals", 1e-2, 0.9)):
        c0, c1 = res[0]["canonical"][key], res[1]["canonical"][key]
        o0, o1 = res[0]["observation"][key], res[1]["observation"][key]
        assert close(c0, c1, tol, frac), key                     # canonical: blind to the head's rotation
        assert (o0 - c0).abs().max().item() <= 1e-4, key         # identity warp at timestep 0
        assert close(o1, o0 @ Rd, tol, frac), key                # observation: n1 = R^T n0
        assert not close(o1, o0, 0.02, 0.5), key
