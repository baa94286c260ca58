"""Mesh export on the GPU (nsb_mesh_count / nsb_mesh_emit, ops.extract_mesh, NeRSembleNGPModel.extract_mesh): the kernels
against the numpy oracle on given density grids, the field end to end against the CPU oracle (density, mesh, normals,
colours), a rigid deformation that must rotate the observed mesh, the occupancy grid, and the model surface."""
import numpy as np
import pytest
import torch

import mesh_oracle as mo
from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
             deform_last_scale=2e-2)
WH, WD = 32.0, 7.0
TIME = 1.0 / 3.0


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


def _mesh(sigma, level, box_min, h):
    from nersemble_b200 import ops
    out = ops.marching_tetrahedra(torch.as_tensor(sigma).to(DEV), level, box_min, h)
    return out["vertices"].cpu().numpy(), out["faces"].cpu().numpy()


def _same_mesh(got, want, extent):
    (gv, gf), (wv, wf) = got, want
    assert gf.shape == wf.shape and np.array_equal(gf, wf)
    assert gv.shape == wv.shape
    if len(gv):
        assert np.abs(gv - wv).max() <= 1e-6 * extent, np.abs(gv - wv).max()


def _grids():
    rng = np.random.default_rng(5)
    out = {}
    out["sphere"] = mo.sample_grid(mo.sphere(0.7), 48) + (0.0,)
    out["torus"] = mo.sample_grid(mo.torus(0.55, 0.25), 40) + (0.0,)
    blobs = lambda X, Y, Z: np.maximum(0.3 - np.sqrt((X - 0.45) ** 2 + Y ** 2 + Z ** 2),
                                       0.25 - np.sqrt((X + 0.5) ** 2 + (Y - 0.2) ** 2 + Z ** 2))
    out["two_blobs"] = mo.sample_grid(blobs, 36) + (0.0,)
    noise = rng.standard_normal((40, 48, 64)).astype(np.float32)          # nz, ny, nx: a non-cubic grid
    out["noise"] = (noise, [-1.0, -0.5, 0.25], [0.03, 0.02, 0.05], 0.1)
    quant = (np.round(rng.standard_normal((20, 24, 28)) * 2) / 2).astype(np.float32)     # many values exactly at the level
    out["equal_to_level"] = (quant, [0.0, 0.0, 0.0], [1.0, 1.0, 1.0], 0.5)
    out["all_below"] = (np.zeros((8, 9, 10), np.float32), [0.0] * 3, [0.1] * 3, 0.5)
    out["all_above"] = (np.ones((8, 9, 10), np.float32), [0.0] * 3, [0.1] * 3, 0.5)
    return out


GRIDS = _grids()


@pytest.mark.parametrize("name", list(GRIDS))
def test_kernel_matches_the_oracle_on_given_grids(name):
    sigma, box_min, h, level = GRIDS[name]
    want = mo.marching_tetrahedra(sigma, level, box_min, h)
    extent = max(h[k] * (sigma.shape[2 - k] - 1) for k in range(3))
    got = _mesh(sigma, level, box_min, h)
    _same_mesh(got, want, extent)
    again = _mesh(sigma, level, box_min, h)
    assert np.array_equal(got[0].view(np.uint32), again[0].view(np.uint32)) and np.array_equal(got[1], again[1])
    if name.startswith("all_"):
        assert len(got[0]) == 0 and len(got[1]) == 0
    else:
        assert len(got[1]) > 100
    if name in ("sphere", "torus", "two_blobs"):
        edges, uses, n_fwd = mo.edge_use(got[1])
        assert (uses == 2).all() and (n_fwd == 1).all() and mo.signed_volume(*got) > 0


def test_kernel_tile_edges():
    """Grids whose point count is 1 below, at and 1 above a multiple of the tile, and one of several thousand tiles
    (the scan's per-thread runs), give the oracle's mesh."""
    rng = np.random.default_rng(9)
    for shape in ((4, 16, 16), (2, 2, 255), (2, 2, 256), (2, 3, 171), (48, 100, 130)):
        sigma = rng.standard_normal(shape).astype(np.float32)
        h = [0.1, 0.2, 0.3]
        _same_mesh(_mesh(sigma, 0.2, [0.0] * 3, h), mo.marching_tetrahedra(sigma, 0.2, [0.0] * 3, h), 40.0)


def _oracle_density(P, pos, space):
    ts = pl.timesteps_from_times(torch.full((pos.shape[0],), TIME), P.n_timesteps)
    out = []
    for i in range(0, pos.shape[0], 4096):
        p, t = pos[i:i + 4096], ts[i:i + 4096]
        if space == "observation":
            out.append(pl.field_density_fn(P, p, torch.full((p.shape[0],), TIME), WH, WD)[:, 0])
        else:       # without the deformation the kernels blend the table lines with fp16 member weights
            code, window = pl.blend_code(P, P.time_emb[t], WH)
            out.append(pl.field_density(P, p, (code * window[None, :]).half().float(), None)[0][:, 0])
    return torch.cat(out)


@pytest.fixture(scope="module")
def field():
    P = oracle_params(KNOBS)
    return P, native_from_oracle(P, DEV)


@pytest.mark.parametrize("space", ["observation", "canonical"])
def test_field_end_to_end_matches_the_oracle(field, space):
    """Density grid against the oracle density (sigma rtol 5e-3); the kernel's mesh of that grid is the oracle's mesh of
    the same grid; vertex normals at the bars of the normals tests; colours seen along -normal at rgb atol 2e-3."""
    from nersemble_b200 import ops
    from normals_oracle import field_normals as canonical_normals
    from deform_jacobian_oracle import observation_normals
    P, NP = field
    res = (30, 24, 28)
    g = ops.density_grid(NP, time=TIME, resolution=res, space=space, window_hash=WH, window_deform=WD)
    sigma = g["sigma"].cpu()
    axes = [mo.grid_positions(n, g["box_min"][k], g["h"][k]) for k, n in enumerate(res)]
    Z, Y, X = np.meshgrid(axes[2], axes[1], axes[0], indexing="ij")
    pos = torch.from_numpy(np.stack([X, Y, Z], -1).reshape(-1, 3))
    want = _oracle_density(P, pos, space).reshape(sigma.shape)
    for v in (want[0], want[-1], want[:, 0], want[:, -1], want[:, :, 0], want[:, :, -1]):
        v.zero_()
    torch.testing.assert_close(sigma, want, rtol=5e-3, atol=1e-5)
    level = float(sigma[1:-1, 1:-1, 1:-1].median())
    mesh = ops.extract_mesh(NP, time=TIME, level=level, resolution=res, space=space, window_hash=WH, window_deform=WD)
    got = {k: v.cpu() for k, v in mesh.items()}
    extent = max(NP.aabb_list[3 + k] - NP.aabb_list[k] for k in range(3))
    _same_mesh((got["vertices"].numpy(), got["faces"].numpy()),
               mo.marching_tetrahedra(sigma.numpy(), level, g["box_min"], g["h"]), extent)
    assert got["faces"].shape[0] > 1000
    v = got["vertices"]
    V = v.shape[0]
    ts = pl.timesteps_from_times(torch.full((V,), TIME), P.n_timesteps)
    if space == "observation":
        off = ops.field_forward(NP, window_hash=WH, window_deform=WD, positions=v.to(DEV), sample_times=torch.full((V,), TIME, device=DEV),
                                uniform_time=TIME, want=("offsets",))["offsets"].cpu()
        wn, grad, sel = observation_normals(P, v, P.time_emb_deform[ts], P.time_emb[ts], WH, WD, world_space=True, offsets=off)
        assert (got["normals"][~sel] == 0).all()
    else:
        wn, grad = canonical_normals(P, v, P.time_emb[ts], WH, world_space=True, blend_fp16=True)
        sel = torch.ones(V, dtype=torch.bool)
    gn = grad.norm(dim=-1)
    keep = sel & (gn >= 1e-3 * gn[sel].median())
    ang = torch.rad2deg(torch.acos((got["normals"][keep] * wn[keep]).sum(-1).clamp(-1, 1)))
    # the normals tests' bars are >= 99.9 % within 1 degree and all within 5 degrees over 3000 samples; over the ~60 000
    # vertices here the observation space shows a tail of at most 1 in 10 000 beyond 5 degrees (measured: 1 vertex at 47)
    n_far = int((ang > 5.0).sum())
    print(f"{space} normals: {V} vertices, {(ang <= 1.0).float().mean().item():.5f} within 1 degree, {n_far} beyond 5, "
          f"worst {ang.max().item():.2f}")
    assert keep.sum() > 0.9 * V and (ang <= 1.0).float().mean() >= 0.999, (ang.max(), keep.sum(), V)
    assert n_far <= (0 if space == "canonical" else max(1, V // 10000)), n_far
    # colours: the oracle's rgb for the same view directions
    dirs = torch.where((got["normals"] == 0).all(-1, keepdim=True), torch.tensor(ops.MESH_FALLBACK_DIRECTION), -got["normals"])
    if space == "observation":
        xw = v + pl.compute_offsets(P, v, P.time_emb_deform[ts], WD)
        _, geo = pl.field_density(P, xw, P.time_emb[ts], WH)
    else:
        code, window = pl.blend_code(P, P.time_emb[ts], WH)
        _, geo = pl.field_density(P, v, (code * window[None, :]).half().float(), None)
    rgb = pl.field_rgb(P, dirs, geo)
    torch.testing.assert_close(got["colours"], rgb, rtol=0, atol=2e-3)


def _rotation(r):
    th = (r * r).sum().clamp_min(1e-4).sqrt()
    K = torch.tensor([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    return torch.eye(3) + (th.sin() / th) * K + ((1 - th.cos()) / th ** 2) * (K @ K)


def _nearest_distance(a, b):
    """Distance from each row of a to the nearest row of b (on the GPU, in chunks)."""
    a, b = a.to(DEV), b.to(DEV)
    return torch.cat([torch.cdist(a[i:i + 2048], b).min(1).values for i in range(0, a.shape[0], 2048)]).cpu()


def test_observation_mesh_is_the_rotated_canonical_mesh():
    """A pure rotation about the box origin (unit box, x = R p): the observed surface is R^T times the canonical one.  Over
    the interior of the box (away from where the rotation carries points out of it), the symmetric Chamfer distance
    between the observation mesh and the rotated canonical mesh is below one voxel, and the normals turn with them."""
    from nersemble_b200 import ops
    r = (0.05, -0.08, 0.06)     # moves the inner region by up to 6 voxels, and keeps its warped positions inside the box
    P = pl.random_params(n_timesteps=2, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
                         aabb=((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)))
    for w, b in zip(P.deform_w, P.deform_b):
        w.zero_(); b.zero_()
    P.r_b.copy_(torch.tensor(r))
    P.tables[int(P.levels.offset[3]):] = 0        # a smooth field (levels of resolution <= 33) that a 64^3 grid resolves
    NP = native_from_oracle(P, DEV)
    can_g = ops.density_grid(NP, time=0.0, resolution=64, space="canonical", window_hash=WH)["sigma"]
    level = float(can_g[16:48, 16:48, 16:48].median())
    kw = dict(time=0.0, level=level, resolution=64, window_hash=WH, window_deform=WD)
    can = {k: v.cpu() for k, v in ops.extract_mesh(NP, space="canonical", normals=False, colours=False, **kw).items()}
    obs = {k: v.cpu() for k, v in ops.extract_mesh(NP, space="observation", colours=False, **kw).items()}
    R = _rotation(torch.tensor(r))
    rot = can["vertices"] @ R              # rows: R^T x
    voxel = 1.0 / 63
    inner = lambda p: ((p > 0.3) & (p < 0.7)).all(-1)
    a = obs["vertices"][inner(obs["vertices"])]
    b = rot[inner(rot)]
    assert a.shape[0] > 500 and b.shape[0] > 500
    da = _nearest_distance(a, rot)
    db = _nearest_distance(b, obs["vertices"])
    chamfer = 0.5 * (da.mean() + db.mean())
    print(f"rigid rotation: chamfer {chamfer / voxel:.3f} voxel, worst {max(da.max(), db.max()) / voxel:.2f} voxel")
    assert chamfer < voxel
    # normals: n_obs(p) = R^T n_can(R p), with the canonical normals taken at the rotated vertices themselves
    n_obs = obs["normals"][inner(obs["vertices"])]
    q = (a @ R.T).to(DEV)                 # rows: R p
    n_at = ops.field_normals(NP, offsets=torch.zeros_like(q), positions=q, sample_times=torch.zeros(q.shape[0], device=DEV),
                             uniform_time=0.0, window_hash=WH, world_space=True)["normals"].cpu()
    cos = (n_obs * (n_at @ R)).sum(-1)
    print(f"rigid rotation: normals cos median {cos.median().item():.6f}, {(cos > 0.999).float().mean().item():.4f} above 0.999")
    assert cos.median() > 0.9999 and (cos > 0.999).float().mean() > 0.99, (cos.median(), (cos > 0.999).float().mean())
    assert (n_obs * n_at).sum(-1).median() < 0.999           # the normals did turn (by about 6 degrees)


def test_cleared_occupancy_cells_give_no_surface(field):
    """With the occupancy cells of the lower half in x cleared, no vertex lies more than one voxel inside that half; without
    the occupancy grid there are vertices deep inside it."""
    from nersemble_b200 import ops
    P, NP = field
    res = 32
    binaries = torch.ones((1, res, res, res), dtype=torch.bool, device=DEV)
    binaries[0, : res // 2] = False
    aabbs = torch.tensor([NP.aabb_list], device=DEV)
    g = ops.density_grid(NP, time=TIME, resolution=48, window_hash=WH, window_deform=WD)
    level = float(g["sigma"][1:-1, 1:-1, 1:-1].median())
    kw = dict(time=TIME, level=level, resolution=48, window_hash=WH, window_deform=WD, normals=False, colours=False)
    full = ops.extract_mesh(NP, **kw)["vertices"].cpu()
    part = ops.extract_mesh(NP, binaries=binaries, aabbs=aabbs, **kw)["vertices"].cpu()
    x_mid = 0.5 * (NP.aabb_list[0] + NP.aabb_list[3])
    voxel = g["h"][0]
    assert (full[:, 0] < x_mid - 4 * voxel).sum() > 100
    assert part.shape[0] > 100 and (part[:, 0] >= x_mid - voxel * (1 + 1e-4)).all(), part[:, 0].min()


def test_model_extract_mesh_and_ply(tmp_path):
    from nersemble_b200 import ops
    from nersemble_b200.mesh import Mesh
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P = oracle_params(KNOBS)
    m = make_model(T=4, log2T=14)
    load_oracle_params_into(m, P)
    m = m.to(DEV).eval()
    occ = blob_grid(5)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    empty = m.extract_mesh(1, resolution=24, respect_occupancy=False, level=1e30)
    assert empty.vertices.shape == (0, 3) and empty.faces.shape == (0, 3)
    default = m.extract_mesh(1, resolution=24)           # level ln 2 / render_step_size
    assert default.vertices.dtype == np.float32 and default.faces.dtype == np.int32
    wh, wd = m._windows()
    g = ops.density_grid(m.native_params(), time=1.0 / 3.0, resolution=40, window_hash=wh, window_deform=wd, **m._blend_opts())
    level = float(g["sigma"][1:-1, 1:-1, 1:-1].median())
    mesh = m.extract_mesh(1, resolution=40, level=level, space="canonical", respect_occupancy=False)
    obs = m.extract_mesh(1, resolution=40, level=level, respect_occupancy=False)
    assert len(mesh.faces) > 100 and len(obs.faces) > 100
    for mm in (mesh, obs):
        assert mm.normals.shape == mm.vertices.shape and mm.colours.shape == mm.vertices.shape
        assert np.isfinite(mm.colours).all() and (mm.colours >= 0).all() and (mm.colours <= 1).all()
    path = str(tmp_path / "head.ply")
    obs.save_ply(path)
    back = Mesh.load_ply(path)
    assert np.array_equal(back.vertices, obs.vertices) and np.array_equal(back.faces, obs.faces)
