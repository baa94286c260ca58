"""Per-timestep blended tables (NativeParams.timestep_tables): inference calls whose samples carry mixed timesteps
gather one float2 per corner from a stack of every timestep's member-blended table instead of the 128 B line of all
32 members.  The stack's slices are the single-frame tables bit for bit; renders on the stack match the per-sample line
gather and the CPU oracle within the north-star tolerance; T > 32 keeps the line gather; in-place table updates rebuild
the cached stack."""
import pytest
import torch

from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp import nerfacc_cpu
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


def _rays(R, seed):
    from oracle.gen_golden import ring_rays
    o, d, t, _ = ring_rays(R, seed)
    return o, d, t


@pytest.mark.parametrize("w_hash", [1, 1.5, 32.0])
def test_stack_slices_equal_the_frame_tables(trained, w_hash):
    _, NP = trained
    T = NP.n_timesteps
    stack = NP.timestep_tables(w_hash, True, True)
    assert stack.shape == (T, NP.tables.shape[0], 2)
    for t in range(T):
        assert torch.equal(stack[t], NP.frame_table(t / (T - 1), w_hash, True, True)), t


def _render(NP, o, d, t, sampler, occ, aabbs, **kw):
    from nersemble_b200 import ops
    if sampler == "fixed":
        return ops.render_rays(NP, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=50,
                               near_plane=0.2, step=0.011, **kw)
    R = o.shape[0]
    return ops.render_rays(NP, o, d, t, window_hash=32.0, window_deform=7.0, sampler="occupancy",
                           near_planes=torch.full((R,), 0.2, device=DEV), far_planes=torch.full((R,), 1e3, device=DEV),
                           binaries=occ, aabbs=aabbs, step=0.011, **kw)


@pytest.mark.parametrize("sampler", ["fixed", "occupancy"])
def test_mixed_timestep_render_on_the_stack(trained, sampler):
    from oracle.gen_golden import blob_grid
    P, NP = trained
    R = 60
    o, d, times = _rays(R, 3)
    assert len(set((times[:, 0] * (NP.n_timesteps - 1)).round().tolist())) == NP.n_timesteps     # every timestep occurs
    occ, aabbs = blob_grid(5)[None].to(DEV), P.aabb.reshape(1, 6).to(DEV)
    args = (o.to(DEV), d.to(DEV), times.to(DEV), sampler, occ, aabbs)
    NP._stack = None
    got = _render(NP, *args)
    assert NP._stack is not None                                  # the render gathered the stack
    line = _render(NP, *args, line_gather=True)
    assert torch.equal(got["packed_info"], line["packed_info"])
    pk, pl_ = got.packed(), line.packed()
    for k in ("t_starts", "t_ends", "ray_indices", "offsets"):      # the march and the deformation do not change
        assert torch.equal(pk[k], pl_[k]), k
    assert pk["t_starts"].shape[0] > 1000
    ts, te, ri = pk["t_starts"].cpu(), pk["t_ends"].cpu(), pk["ray_indices"].cpu().long()
    with torch.no_grad():
        want = pl.render(P, o, d, times, ts, te, ri, window_hash=32.0, window_deform=7.0, training=False)
    for ref in (want, {k: v.cpu() for k, v in line.items() if torch.is_tensor(v)}):
        assert (got["rgb"].cpu() - ref["rgb"]).norm(dim=-1).max() < 1e-3
        torch.testing.assert_close(got["accumulation"].cpu(), ref["accumulation"], rtol=0, atol=1e-3)
        torch.testing.assert_close(got["depth"].cpu(), ref["depth"], rtol=1e-3, atol=1e-3)
    assert torch.equal(got["num_samples_per_ray"].cpu(), nerfacc_cpu.pack_info(ri, R)[:, 1])


def test_field_forward_on_the_stack_matches_the_line_gather(trained):
    """field_forward (the three-kernel path of render_packed) takes the same stack: same deformation bit for bit, the
    blend differs by rounding only."""
    from nersemble_b200 import ops
    P, NP = trained
    R = 40
    o, d, times = _rays(R, 7)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 50, 0.011, near=0.2)
    kw = dict(origins=o.to(DEV), directions=d.to(DEV), ray_times=times.to(DEV), t_starts=ts.to(DEV), t_ends=te.to(DEV),
              ray_indices=ri.to(DEV), window_hash=32.0, window_deform=7.0)
    stack = ops.field_forward(NP, **kw)
    line = ops.field_forward(NP, line_gather=True, **kw)
    assert torch.equal(stack["offsets"], line["offsets"])
    torch.testing.assert_close(stack["sigma"], line["sigma"], rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(stack["rgb"], line["rgb"], rtol=0, atol=2e-3)


def test_more_than_32_timesteps_keep_the_line_gather():
    """T = 40: the stack would be 2.5x the line tables -- none is built, and the render is the line gather's."""
    P = oracle_params(dict(KNOBS, n_timesteps=40))
    NP = native_from_oracle(P, DEV)
    assert NP.timestep_tables(32.0, True, True) is None
    o, d, times = _rays(30, 4)
    args = (o.to(DEV), d.to(DEV), times.to(DEV), "fixed", None, None)
    got = _render(NP, *args)
    line = _render(NP, *args, line_gather=True)
    assert getattr(NP, "_stack", None) is None
    for k in ("rgb", "accumulation", "depth", "deformation"):
        assert torch.equal(got[k], line[k]), k


def test_in_place_table_update_rebuilds_the_stack():
    P = oracle_params(KNOBS)
    NP = native_from_oracle(P, DEV)
    o, d, times = _rays(30, 6)
    args = (o.to(DEV), d.to(DEV), times.to(DEV), "fixed", None, None)
    before = NP.timestep_tables(32.0, True, True).clone()
    a = _render(NP, *args)["rgb"].clone()
    NP.tables.mul_(0.5)                                           # an optimiser step: same storage, new version
    after = NP.timestep_tables(32.0, True, True)
    torch.testing.assert_close(after, before * 0.5, rtol=1e-5, atol=1e-6)
    b = _render(NP, *args)["rgb"]
    line = _render(NP, *args, line_gather=True)["rgb"]
    assert (b - line).norm(dim=-1).max() < 1e-3 and (b - a).abs().max() > 1e-3
