"""The wgmma tensor role (two warpgroups of 64 rows each) at the edges of its tile schedule: a last tile of 1, 63, 64 or
65 rows (warpgroup 1 with only padding rows, or one row), fewer tiles than SMs, one tile per CTA, and CTAs with no
tile at all in the one-launch render kernel.  Each case is checked against the mma.sync role and the CPU oracle."""
import pytest
import torch

from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp import nerfacc_cpu
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TRAINED = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
               deform_last_scale=1e-3)


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@pytest.fixture(scope="module")
def roles():
    P = oracle_params(TRAINED)
    return P, native_from_oracle(P, DEV, tcgen05=True), native_from_oracle(P, DEV, tcgen05=False)


def _packed_samples(P, n):
    """The first n fixed-stride samples of a ring of rays (packed by ray), with the rays and their mixed times."""
    from oracle.gen_golden import ring_rays
    R = n // 40 + 2
    o, d, times, _ = ring_rays(R, 5)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 64, 0.011, near=0.2)
    assert ts.shape[0] >= n
    ts, te, ri = ts[:n], te[:n], ri[:n]
    return o, d, times, ts, te, ri, nerfacc_cpu.pack_info(ri, R)


# full tiles before the ragged one: 0 (a single tile), 5 (6 tiles: fewer than the SMs, one per CTA), 140 (141 tiles: the
# ragged tile is the second of its CTA)
@pytest.mark.parametrize("full_tiles", [0, 5, 140])
@pytest.mark.parametrize("last_rows", [1, 63, 64, 65])
def test_ragged_last_tile_vs_mma_role_and_oracle(roles, full_tiles, last_rows):
    from nersemble_b200 import ops
    P, NP_tc, NP_mma = roles
    n = full_tiles * 128 + last_rows
    o, d, times, ts, te, ri, info = _packed_samples(P, n)
    with torch.no_grad():
        want = pl.render(P, o, d, times, ts, te, ri, window_hash=32.0, window_deform=7.0, training=False)
    args = [x.to(DEV) for x in (o, d, times, ts, te, ri, info)]
    got = {k: v.cpu() for k, v in ops.render_packed(NP_tc, *args, window_hash=32.0, window_deform=7.0, training=False).items()}
    mma = {k: v.cpu() for k, v in ops.render_packed(NP_mma, *args, window_hash=32.0, window_deform=7.0, training=False).items()}
    for ref in (want, mma):
        torch.testing.assert_close(got["offsets"], ref["offsets"], rtol=2e-3, atol=3e-6)
        torch.testing.assert_close(got["density"], ref["density"], rtol=5e-3, atol=1e-5)
        torch.testing.assert_close(got["rgb_samples"], ref["rgb_samples"], rtol=0, atol=2e-3)
        assert (got["rgb"] - ref["rgb"]).norm(dim=-1).max() < 1e-3
        torch.testing.assert_close(got["accumulation"], ref["accumulation"], rtol=0, atol=1e-3)
    assert torch.equal(got["num_samples_per_ray"], want["num_samples_per_ray"])


@pytest.mark.parametrize("n", [1, 63, 64, 65, 132 * 128, 132 * 128 + 65])
def test_sample_based_line_gather_vs_mma_role(roles, n):
    """field_forward on positions with the per-sample line gather (the non-frame-table tc kernel); 132 x 128 samples
    give every CTA of an H100 exactly one tile."""
    from nersemble_b200 import ops
    P, NP_tc, NP_mma = roles
    g = torch.Generator().manual_seed(n)
    lo, hi = P.aabb[0], P.aabb[1]
    pos = (lo + (hi - lo) * torch.rand((n, 3), generator=g)).to(DEV)
    tt = torch.rand((n,), generator=g).to(DEV)
    kw = dict(window_hash=32.0, window_deform=7.0, positions=pos, sample_times=tt, want=("sigma", "rgb", "offsets"),
              line_gather=True)
    got, mma = ops.field_forward(NP_tc, **kw), ops.field_forward(NP_mma, **kw)
    torch.testing.assert_close(got["offsets"], mma["offsets"], rtol=2e-3, atol=3e-6)
    torch.testing.assert_close(got["sigma"], mma["sigma"], rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(got["rgb"], mma["rgb"], rtol=0, atol=2e-3)


@pytest.mark.parametrize("R", [1, 3, 40])
def test_render_kernel_with_idle_ctas_vs_mma_role_and_oracle(roles, R):
    """The one-launch render kernel always runs one CTA per SM: with 1-40 rays of 48 samples most CTAs get no tile."""
    from nersemble_b200 import ops
    from oracle.gen_golden import ring_rays
    P, NP_tc, NP_mma = roles
    o, d, times, _ = ring_rays(R, 11)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 48, 0.011, near=0.2)
    with torch.no_grad():
        want = pl.render(P, o, d, times, ts, te, ri, window_hash=32.0, window_deform=7.0, training=False)
    kw = dict(window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=48, near_plane=0.2, step=0.011)
    got = ops.render_rays(NP_tc, o.to(DEV), d.to(DEV), times.to(DEV), **kw)
    mma = ops.render_rays(NP_mma, o.to(DEV), d.to(DEV), times.to(DEV), **kw)
    for ref in (want["rgb"], mma["rgb"].cpu()):
        assert (got["rgb"].cpu() - ref).norm(dim=-1).max() < 1e-3
    torch.testing.assert_close(got["accumulation"].cpu(), want["accumulation"], rtol=0, atol=1e-3)
