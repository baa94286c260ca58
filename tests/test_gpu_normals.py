"""Surface normals on the GPU (nsb_normals_forward): per-sample normals of the field API and of render samples against
the CPU oracle (autograd of h0 with respect to the masked normalised position, kernel precision), the three gather modes
against each other, the rendered normals channel against the oracle composite, and the plugin surface."""
import pytest
import torch

from conftest import native_from_oracle, oracle_params
from normals_oracle import composite_normals, field_normals as oracle_normals
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
             deform_last_scale=1e-3)


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@pytest.fixture(scope="module")
def trained():
    P = oracle_params(KNOBS)
    return P, native_from_oracle(P, DEV)


def _angles(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Angle in degrees between rows of two unit-vector sets."""
    return torch.rad2deg(torch.acos((a * b).sum(-1).clamp(-1.0, 1.0)))


def _check_angles(got, want, g_ref, what):
    """At least 99.9 % within 1 degree and all within 5 degrees, over samples whose oracle gradient norm is at least
    1e-3 of the median (the direction of a vanishing gradient is noise)."""
    gn = g_ref.norm(dim=-1)
    keep = gn >= 1e-3 * gn.median()
    ang = _angles(got[keep], want[keep])
    assert keep.sum() > 0.9 * keep.numel(), what
    frac = (ang <= 1.0).float().mean().item()
    assert frac >= 0.999 and ang.max().item() <= 5.0, (what, frac, ang.max().item(), int(keep.sum()))


def _rays(R, seed):
    from oracle.gen_golden import ring_rays
    o, d, t, _ = ring_rays(R, seed)
    return o, d, t


def _render(NP, o, d, t, **kw):
    from nersemble_b200 import ops
    return ops.render_rays(NP, o.to(DEV), d.to(DEV), None if t is None else t.to(DEV), window_hash=32.0, window_deform=7.0,
                           sampler="fixed", n_per_ray=48, near_plane=0.2, step=0.1, want_normals=True, **kw)


def _oracle_for_render(P, o, d, t, pk, world_space=True, blend_fp16=False):
    ri = pk["ray_indices"].cpu().long()
    mid = (pk["t_starts"] + pk["t_ends"]).cpu()
    pos = o[ri] + d[ri] * mid[:, None] * 0.5          # the kernels' o + (d * mid) * 0.5
    ts = pl.timesteps_from_times(t[ri], P.n_timesteps) if t is not None else torch.zeros_like(ri)
    off = pk["offsets"].cpu() if "offsets" in pk else None
    return oracle_normals(P, pos, P.time_emb[ts], 32.0, offsets=off, world_space=world_space, blend_fp16=blend_fp16)


def test_field_api_normals_match_the_oracle(trained):
    """Explicit positions with per-sample blend codes (the component field API), a fifth of them outside the box.  The
    line gather rounds the member weights to fp16 (blend_fp16 in the oracle): with fp32 weights about 0.5 % of the
    samples flip a ReLU of mlp_base and their normal turns by up to tens of degrees."""
    from nersemble_b200 import ops
    P, NP = trained
    gen = torch.Generator().manual_seed(11)
    n = 3000
    x = torch.rand((n, 3), generator=gen) * 1.25 - 0.125
    pos = P.aabb[0] + x * (P.aabb[1] - P.aabb[0])
    codes = torch.randn((n, 32), generator=gen) * 0.3
    got = ops.field_normals(NP, window_hash=20.25, positions=pos.to(DEV), sample_blend_codes=codes.to(DEV))["normals"]
    want, g = oracle_normals(P, pos, codes, 20.25, blend_fp16=True)
    sel = ((x > 0) & (x < 1)).all(-1)
    assert 0.3 < sel.float().mean() < 0.8
    out = ~sel     # out-of-box samples: the gradient at the box origin, one direction per code
    assert torch.isfinite(got).all() and (got.norm(dim=-1) - 1).abs().max() < 1e-5
    _check_angles(got.cpu(), want, g, "field API")
    _check_angles(got.cpu()[out], want[out], g[out], "field API, outside the box")


@pytest.mark.parametrize("mode", ["stack", "line", "no_deform"])
def test_render_sample_normals_match_the_oracle(trained, mode):
    """Per-sample normals of render samples (world space), mixed timesteps: the timestep stack, the line gather, and
    the line gather without deformation.  The fixed sampler marches past the box exit: out-of-box samples included."""
    P, NP = trained
    o, d, t = _rays(96, 3)
    kw = dict(line_gather=mode != "stack", use_deformation=mode != "no_deform")
    NP._stack = None
    res = _render(NP, o, d, t, **kw)
    assert (NP._stack is not None) == (mode == "stack")
    pk = res.packed()
    want, g = _oracle_for_render(P, o, d, t, pk, blend_fp16=mode != "stack")
    xw = pk["offsets"].cpu() if "offsets" in pk else 0.0
    ri = pk["ray_indices"].cpu().long()
    pn = (o[ri] + d[ri] * (pk["t_starts"] + pk["t_ends"]).cpu()[:, None] * 0.5 + xw - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    assert (~((pn > 0) & (pn < 1)).all(-1)).sum() > 100          # out-of-box samples are part of the comparison
    _check_angles(pk["normals"].cpu(), want, g, mode)


def test_gather_modes_agree(trained):
    """One camera frame (uniform time): the frame table, the timestep stack and the line gather read the same numbers
    up to the blend's rounding; the samples and offsets are the same bits.  Frame table and stack (fp32 member weights)
    agree to the bound.  The line gather rounds the weights to fp16: where it differs from the frame table by more than
    1 degree, the oracle with fp16 weights differs from the oracle with fp32 weights as well (a ReLU of mlp_base
    switches), and the line gather matches the fp16-weight oracle to the bound."""
    P, NP = trained
    o, d, _ = _rays(96, 5)
    t = torch.full((96, 1), 2.0 / 3.0)
    frame = _render(NP, o, d, t, uniform_time=2.0 / 3.0)
    stack = _render(NP, o, d, t)
    line = _render(NP, o, d, t, line_gather=True)
    pf, ps, plg = frame.packed(), stack.packed(), line.packed()
    for k in ("t_starts", "offsets"):
        assert torch.equal(pf[k], ps[k]) and torch.equal(pf[k], plg[k]), k
    w32, g = _oracle_for_render(P, o, d, t, pf)
    w16, g16 = _oracle_for_render(P, o, d, t, pf, blend_fp16=True)
    _check_angles(pf["normals"].cpu(), ps["normals"].cpu(), g, "frame/stack")
    _check_angles(pf["normals"].cpu(), w32, g, "frame/oracle")
    _check_angles(plg["normals"].cpu(), w16, g16, "line/oracle fp16 weights")
    off = _angles(plg["normals"].cpu(), pf["normals"].cpu()) > 1.0
    explained = _angles(w16, w32) > 0.5
    keep = g.norm(dim=-1) >= 1e-3 * g.norm(dim=-1).median()
    assert (off & keep & ~explained).float().mean() <= 1e-3, int((off & keep & ~explained).sum())


def test_rendered_normals_match_the_oracle_composite():
    """4096 rays, trained-like tables (table_scale 1e3): the per-ray channel against the oracle's per-sample normals
    composited with the render's weights: L2 <= 1e-2 where the accumulation is at least 0.5, for all but 0.1 % of those
    rays.  The MLP input is the fp16-rounded feature; at this table scale a feature's fp16 rounding can differ with the
    summation order, switch a ReLU of mlp_base and turn one sample's normal.  The composite itself is checked exactly:
    the per-ray output is the composite of the kernel's own per-sample normals."""
    P = oracle_params(dict(KNOBS, table_scale=1e3, time_std_scale=1.0))
    NP = native_from_oracle(P, DEV)
    R = 4096
    o, d, t = _rays(R, 9)
    res = _render(NP, o, d, t)
    pk = res.packed()
    want_s, g_s = _oracle_for_render(P, o, d, t, pk)
    want = composite_normals(want_s, pk["weights"].cpu(), pk["ray_indices"].cpu(), R)
    got = res["normals"].cpu()
    assert got.shape == (R, 3) and torch.isfinite(got).all()
    acc = res["accumulation"].cpu()[:, 0]
    hit = acc >= 0.5
    assert hit.sum() > R // 4, hit.sum()
    err = (got - want)[hit].norm(dim=-1)
    assert (err > 1e-2).float().mean() <= 1e-3, (err.max(), (err > 1e-2).sum(), hit.sum())
    own = composite_normals(pk["normals"].cpu(), pk["weights"].cpu(), pk["ray_indices"].cpu(), R)
    assert (got - own).norm(dim=-1).max() <= 1e-5
    # per sample: the 99.9 % / 1 degree bound holds; a sample beyond 5 degrees must have a ReLU of mlp_base whose
    # pre-activation lies within the fp16 rounding of the features (measured: 2 of 196 608 samples above 1 degree, the
    # worst 8.1 degrees)
    gn = g_s.norm(dim=-1)
    keep = gn >= 1e-3 * gn.median()
    ang = _angles(pk["normals"].cpu(), want_s)
    assert (ang[keep] <= 1.0).float().mean() >= 0.999
    far = torch.nonzero(keep & (ang > 5.0)).reshape(-1)
    if far.numel():
        from normals_oracle import masked_position
        ri = pk["ray_indices"].cpu().long()[far]
        pos = o[ri] + d[ri] * (pk["t_starts"] + pk["t_ends"]).cpu()[far, None] * 0.5
        x = masked_position(P, pos, pk["offsets"].cpu()[far])
        feat = pl.hash_ensemble(P, x, P.time_emb[pl.timesteps_from_times(t[ri], P.n_timesteps)], 32.0)
        w0 = P.base_w[0].half().float()
        pre = feat.half().float() @ w0.t()
        ulp = torch.exp2(torch.floor(torch.log2(feat.abs().clamp_min(6.1e-5))) - 10)      # fp16 spacing at each feature
        assert ((pre.abs() <= ulp @ w0.abs().t()).any(-1)).all(), (far, ang[far])
    assert ((got[hit].norm(dim=-1) - 1).abs() < 1e-4).all()


def test_render_normals_are_sync_free_and_deterministic(trained):
    from nersemble_b200 import ops
    P, NP = trained
    o, d, t = (v.to(DEV) for v in _rays(256, 4))
    kw = dict(window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=64, near_plane=0.2, step=0.02)
    first = ops.render_rays(NP, o, d, t, want_normals=True, **kw)       # warm-up: packs / builds the cached tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = ops.render_rays(NP, o, d, t, want_normals=True, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    plain = ops.render_rays(NP, o, d, t, **kw)
    assert torch.equal(first["normals"], second["normals"])           # bitwise run to run
    assert "normals" not in plain
    for k in ("rgb", "accumulation", "depth", "deformation", "num_samples_per_ray"):
        assert torch.equal(first[k], plain[k]), k


def test_model_render_normals_channel():
    """NeRSembleNGPModel.render_normals: `normals` on every get_outputs path and in get_outputs_for_camera_ray_bundle;
    the other outputs are the same bits and the key set is unchanged with the flag off."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P = oracle_params(KNOBS)
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
    for fused in (True, False):
        m.use_fused_render = fused
        with torch.no_grad():
            m.render_normals = False
            off = m.get_outputs(rb)
            m.render_normals = True
            on = m.get_outputs(rb)
        assert set(on) == set(off) | {"normals"} and "normals" not in off, fused
        assert on["normals"].shape == (R, 3) and torch.isfinite(on["normals"]).all()
        for k in ("rgb", "accumulation", "depth", "deformation"):
            assert torch.equal(on[k], off[k]), (fused, k)
    m.use_fused_render = True
    H, W = 20, 30
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1.5, 1.5, W), indexing="ij")
    cam_o = torch.tensor([0.0, 0.0, 9.0]).expand(H, W, 3).contiguous()
    cam_d = torch.stack([xs, ys, torch.full_like(xs, -9.0)], -1); cam_d = cam_d / cam_d.norm(dim=-1, keepdim=True)
    cam = RayBundle(origins=cam_o.to(DEV), directions=cam_d.to(DEV), pixel_area=torch.ones(H, W, 1, device=DEV),
                    camera_indices=torch.zeros(H, W, 1, dtype=torch.long, device=DEV), times=torch.full((H, W, 1), 0.34, device=DEV))
    m.render_normals = False
    img_off = m.get_outputs_for_camera_ray_bundle(cam)
    m.render_normals = True
    img_on = m.get_outputs_for_camera_ray_bundle(cam)
    assert set(img_on) == set(img_off) | {"normals"} and img_on["normals"].shape == (H, W, 3)
    for k in img_off:
        assert torch.equal(img_on[k], img_off[k]), k
    # training path (differentiable render): normals of the packed samples, the loss graph unchanged
    m.train(); m.sampler.eval()
    out = m.get_outputs(rb)
    assert out["normals"].shape == (R, 3) and out["normals"].grad_fn is None and out["rgb"].grad_fn is not None


def test_field_compute_normals():
    """NeRSembleNeRFactoField.forward(compute_normals=True) with and without autograd: FieldHeadNames.NORMALS against
    the oracle, RGB / DENSITY the same bits as compute_normals=False; get_normals() = the last call's normals."""
    from nersemble_b200.nerfstudio_shim import FieldHeadNames, Frustums, RaySamples
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P = oracle_params(KNOBS)
    m = make_model(T=4, log2T=14)
    load_oracle_params_into(m, P)
    field = m.to(DEV).field
    gen = torch.Generator().manual_seed(2)
    n = 1000
    x = torch.rand((n, 3), generator=gen) * 1.1 - 0.05
    pos = P.aabb[0] + x * (P.aabb[1] - P.aabb[0])
    dirs = torch.nn.functional.normalize(torch.randn((n, 3), generator=gen), dim=-1)
    codes = torch.randn((n, 32), generator=gen) * 0.3
    rs = RaySamples(frustums=Frustums(origins=pos.to(DEV), directions=dirs.to(DEV), starts=torch.zeros(n, 1, device=DEV),
                                      ends=torch.zeros(n, 1, device=DEV), pixel_area=torch.ones(n, 1, device=DEV)),
                    camera_indices=torch.zeros(n, 1, dtype=torch.long, device=DEV))
    rs.metadata = {"time_codes": codes.to(DEV)}
    want, g = oracle_normals(P, pos, codes, 16.0, blend_fp16=True)
    with torch.no_grad():
        plain = field(rs, window_hash_encodings=16.0)
        got = field(rs, compute_normals=True, window_hash_encodings=16.0)
    for k in (FieldHeadNames.RGB, FieldHeadNames.DENSITY):
        assert torch.equal(got[k], plain[k]), k
    _check_angles(got[FieldHeadNames.NORMALS].cpu(), want, g, "field forward")
    assert torch.equal(field.get_normals(), got[FieldHeadNames.NORMALS])
    with torch.enable_grad():
        out = field(rs, compute_normals=True, window_hash_encodings=16.0)
        assert out[FieldHeadNames.DENSITY].grad_fn is not None and out[FieldHeadNames.NORMALS].grad_fn is None
    assert torch.equal(out[FieldHeadNames.NORMALS], got[FieldHeadNames.NORMALS])
    torch.testing.assert_close(out[FieldHeadNames.RGB], plain[FieldHeadNames.RGB], rtol=0, atol=0)
