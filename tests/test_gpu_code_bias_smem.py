"""The per-timestep code-bias rows of deformation layers 0 and 4 in the wgmma kernels: staged in shared memory (one
swizzled 1 KB row pair per timestep) for up to 32 timesteps, read from the global table above that.  Every timestep
appears in each batch, and the warp codes are large, so a row read for the wrong timestep moves the offsets far outside
the tolerances.  Each case is checked against the mma.sync role."""
import functools

import pytest
import torch

from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CAP = 32        # kTcCodeBiasRows in nsb_field.cu: the most timesteps staged in shared memory
WIN = dict(window_hash=32.0, window_deform=7.0)


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@functools.lru_cache(maxsize=1)
def _roles(T):
    P = oracle_params(dict(seed=20240611, n_timesteps=T, log2_hashmap_size=14, table_scale=0.5, time_std_scale=400.0,
                           deform_last_scale=1e-3))
    return P, native_from_oracle(P, DEV, tcgen05=True), native_from_oracle(P, DEV, tcgen05=False)


def _rays(T, per_ts=3):
    """per_ts rays per timestep, in shuffled order, each at the exact time of its timestep."""
    from oracle.gen_golden import ring_rays
    R = per_ts * T + 5
    o, d, _, _ = ring_rays(R, 31)
    g = torch.Generator().manual_seed(T)
    ts = (torch.arange(R) % T)[torch.randperm(R, generator=g)]
    times = (ts.float() / max(T - 1, 1)).reshape(R, 1)
    return o, d, times


def _close(got, ref):
    torch.testing.assert_close(got["offsets"], ref["offsets"], rtol=2e-3, atol=3e-6)
    torch.testing.assert_close(got["sigma"], ref["sigma"], rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(got["rgb"], ref["rgb"], rtol=0, atol=2e-3)


@pytest.mark.parametrize("T", [1, 24, CAP, CAP + 1])
def test_fused_render_vs_mma_role(T):
    """The one-launch render (fixed march, per-ray times: the timestep-stack kernel, or the per-sample blend above 32)."""
    from nersemble_b200 import ops
    P, NP_tc, NP_mma = _roles(T)
    o, d, times = (x.to(DEV) for x in _rays(T))
    kw = dict(WIN, sampler="fixed", n_per_ray=48, near_plane=0.2, step=0.011)
    got = ops.render_rays(NP_tc, o, d, times, **kw).packed()
    mma = ops.render_rays(NP_mma, o, d, times, **kw).packed()
    assert torch.equal(got["ray_indices"], mma["ray_indices"])
    _close(got, mma)


@pytest.mark.parametrize("T", [1, 24, CAP, CAP + 1])
def test_field_forward_vs_mma_role(T):
    """field_forward on ray samples: per-ray times (every timestep in the batch), and uniform_time for the first, a
    middle and the last timestep (the single frame-table kernel)."""
    from nersemble_b200 import ops
    P, NP_tc, NP_mma = _roles(T)
    o, d, times = _rays(T)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 48, 0.011, near=0.2)
    base = dict(WIN, want=("sigma", "rgb", "offsets"), origins=o.to(DEV), directions=d.to(DEV), t_starts=ts.to(DEV),
                t_ends=te.to(DEV), ray_indices=ri.to(DEV))
    _close(ops.field_forward(NP_tc, ray_times=times.to(DEV), **base), ops.field_forward(NP_mma, ray_times=times.to(DEV), **base))
    for t in sorted({0, T // 2, T - 1}):
        u = t / max(T - 1, 1)
        tu = torch.full_like(times, u).to(DEV)
        _close(ops.field_forward(NP_tc, ray_times=tu, uniform_time=u, **base),
               ops.field_forward(NP_mma, ray_times=tu, uniform_time=u, **base))


def test_wrong_timestep_is_detected():
    """The tolerances above separate neighbouring timesteps: shifting every ray by one timestep moves the offsets."""
    from nersemble_b200 import ops
    T = 24
    P, NP_tc, _ = _roles(T)
    o, d, times = _rays(T)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 48, 0.011, near=0.2)
    base = dict(WIN, want=("offsets",), origins=o.to(DEV), directions=d.to(DEV), t_starts=ts.to(DEV), t_ends=te.to(DEV),
                ray_indices=ri.to(DEV))
    a = ops.field_forward(NP_tc, ray_times=times.to(DEV), **base)["offsets"]
    shifted = torch.remainder(times * (T - 1) + 1, T) / (T - 1)
    b = ops.field_forward(NP_tc, ray_times=shifted.to(DEV), **base)["offsets"]
    with pytest.raises(AssertionError):
        torch.testing.assert_close(a, b, rtol=2e-3, atol=3e-6)
