"""CPU tests of rendering between captured timesteps (DESIGN 4.2g): the time rule ops.time_lerp against a float64
restatement, the Python argument checks, the host checks of nsb_render_forward_interp, its ctypes binding, and the spill
budget of the new render_kernel_tc_lerp instantiations."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT
from nersemble_b200 import _lib, ops

DUMMY = 0x10000      # non-null, never dereferenced: every call below is rejected on the host


def _rule64(t, T):
    """float64 restatement of the rule: u = clamp(fl32(t (T - 1)), 0, T - 1), snapped within 2^-10 to the integer."""
    with np.errstate(invalid="ignore"):
        u = float(np.float32(np.float32(t) * np.float32(T - 1)))    # the kernels' one fp32 product
    u = 0.0 if math.isnan(u) else min(max(u, 0.0), float(T - 1))
    if abs(u - round(u)) <= 2.0 ** -10:
        u = float(round(u))
    i0 = min(int(math.floor(u)), T - 1)
    return i0, min(i0 + 1, T - 1), u - i0


def test_time_lerp_matches_the_float64_rule_and_clamps():
    assert ops.TIME_SNAP == 2.0 ** -10 and ops.TIME_INTERPOLATIONS == ("nearest", "linear")
    for t in (-1.0, -1e-9, 0.0, 1.0, 1.0 + 1e-6, 7.5, float("inf"), float("-inf"), float("nan")):
        for T in (1, 2, 5, 24):
            assert ops.time_lerp(t, T) == _rule64(t, T), (t, T)
    assert ops.time_lerp(0.37, 1) == (0, 0, 0.0)           # T = 1: every time is row 0
    assert ops.time_lerp(0.25, 2) == (0, 1, 0.25)
    assert ops.time_lerp(1.0, 2) == (1, 1, 0.0)
    g = np.random.default_rng(0)
    for T in (2, 3, 24, 48, 2000):
        for t in g.random(300):
            got = ops.time_lerp(float(t), T)
            assert got == _rule64(float(t), T), (t, T)
            assert 0 <= got[2] < 1 and got[1] == min(got[0] + 1, T - 1)
    with pytest.raises(ValueError, match="n_timesteps"):
        ops.time_lerp(0.5, 0)


@pytest.mark.parametrize("T", [2, 3, 7, 24, 33, 100, 1000, 2000, 4096])
def test_captured_times_snap_to_their_timestep(T):
    """float32(k) / (T - 1) and float32(k / (T - 1)) land a few ulp off k after the kernels' product; both snap to k,
    the timestep the nearest path's __float2int_rn picks."""
    for k in range(T):
        for t in (float(np.float32(np.float32(k) / np.float32(T - 1))), float(np.float32(k / (T - 1)))):
            assert ops.time_lerp(t, T) == (k, min(k + 1, T - 1), 0.0), (k, T, t)
            assert int(np.rint(np.float32(t) * np.float32(T - 1))) == k


@pytest.mark.parametrize("T", [2, 5, 24, 48])
def test_lam_is_monotone_between_timesteps(T):
    ts = np.linspace(0.0, 1.0, 20001, dtype=np.float32)
    u = np.array([(lambda r: r[0] + r[2])(ops.time_lerp(float(t), T)) for t in ts])
    assert np.all(np.diff(u) >= 0), "u(t) must not decrease"
    assert u[0] == 0 and u[-1] == T - 1


def test_device_rule_mirrors_the_host_rule():
    g = torch.Generator().manual_seed(1)
    for T in (1, 2, 24, 48, 2000):
        t = torch.cat([torch.rand(500, generator=g), torch.arange(T, dtype=torch.float32) / max(T - 1, 1),
                       torch.tensor([-0.5, 1.5, float("nan")])])
        i0, i1, lam = ops.time_lerp_rows(t, T)
        want = [ops.time_lerp(float(x), T) for x in t]
        assert i0.tolist() == [w[0] for w in want] and i1.tolist() == [w[1] for w in want]
        assert lam.tolist() == [w[2] for w in want]


def test_lerp_is_fmaf():
    """_lerp_f32 rounds fmaf(lam, b - a, a) once; at lam = 0 it is a."""
    g = torch.Generator().manual_seed(2)
    a, b = torch.randn(4096, generator=g), torch.randn(4096, generator=g) * 3
    for lam in (0.0, 0.25, 0.3333333432674408, 0.999):
        got = ops._lerp_f32(a, b, lam)
        want = torch.tensor([np.float32(np.float64(lam) * np.float64(np.float32(y - x)) + np.float64(x))
                             for x, y in zip(a.numpy(), b.numpy())])
        assert torch.equal(got, want)
    assert torch.equal(ops._lerp_f32(a, b, 0.0), a)


def test_python_arguments_are_validated_before_any_device_call():
    # None parameters / tensors: a check that came after any device work would fail differently
    with pytest.raises(ValueError, match="time_interpolation"):
        ops.render_rays(None, None, None, None, time_interpolation="cubic")
    P = ops.NativeParams(None, None, None, None, None, torch.zeros(6), {"n_levels": 0}, 4)
    for kw, match in ((dict(use_deformation=False), "use_deformation=False"),
                      (dict(want_normals=True), "want_normals=True"),
                      (dict(), "non-wgmma")):
        with pytest.raises(NotImplementedError, match=match):
            ops.render_rays(P, None, None, None, time_interpolation="linear", **kw)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib.load()


def _params(**over):
    p = _lib.FieldParams()
    for name, _ in _lib.FieldParams._fields_:
        if name not in ("frame_table", "frame_stride", "n_timesteps", "aabb", "levels"):
            setattr(p, name, DUMMY)
    p.n_timesteps = 4
    p.levels.n_levels = _lib.MAX_LEVELS
    for l in range(_lib.MAX_LEVELS):
        p.levels.offset[l], p.levels.entries[l] = 1024 * l, 1024
    for k in range(3):
        p.aabb[3 + k] = 1.0
    for k, v in over.items():
        setattr(p, k, v)
    return p


def _args(**over):
    a = _lib.RenderArgs()
    for name, ty in _lib.RenderArgs._fields_:
        if ty is C.c_void_p and name not in ("ray_times", "near_planes", "far_planes", "binaries", "aabbs", "march_scratch"):
            setattr(a, name, DUMMY)
    a.n_rays, a.sampler, a.n_per_ray, a.capacity = 64, 0, 4, 256
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_entry_point_rejects_bad_inputs_on_the_host(lib):
    """The checks of nsb_render_forward and the linear-only ones run before any CUDA call and name the entry point."""
    def expect(p, o, a, message):
        rc = lib.nsb_render_forward_interp(None if p is None else C.byref(p), None if o is None else C.byref(o),
                                           None if a is None else C.byref(a), None)
        err = lib.nsb_last_error().decode()
        assert rc != 0 and err == f"nsb_render_forward_interp: {message}", err

    opts = ops.make_opts(None, None, True, True)
    no_def = ops.make_opts(None, None, False, True)
    expect(None, opts, _args(), "null argument")
    expect(_params(), None, _args(), "null argument")
    expect(_params(), opts, None, "null argument")
    expect(_params(n_timesteps=0), opts, _args(), "n_timesteps < 1")
    expect(_params(frame_stride=-1), opts, _args(), "frame_stride out of range")
    expect(_params(), opts, _args(out_rgb=None), "null buffer")
    expect(_params(tables=None), opts, _args(), "tables/field_packed/blend_codes missing")
    expect(_params(deform_code_bias=None), opts, _args(), "deformation parameters missing")
    expect(_params(), opts, _args(capacity=0), "capacity <= 0")
    expect(_params(), opts, _args(capacity=100), "capacity < n_rays * n_per_ray")
    expect(_params(), opts, _args(sampler=1), "occupancy sampler arguments")
    expect(_params(), opts, _args(sampler=7), "unknown sampler")
    expect(_params(), no_def, _args(offsets=None), "linear time needs the deformation field (use_deformation)")
    expect(_params(deform_packed_umma=None), opts, _args(), "linear time needs the wgmma deformation weights (deform_packed_umma)")
    stack = "the frame table must be a timestep stack whose frame_stride covers every level's entries"
    expect(_params(frame_table=DUMMY, frame_stride=0), opts, _args(), stack)
    expect(_params(frame_table=DUMMY, frame_stride=16 * 1024 - 1), opts, _args(), stack)
    # no rays: nothing to check or launch
    assert lib.nsb_render_forward_interp(C.byref(_params()), C.byref(opts), C.byref(_args(n_rays=0)), None) == 0


def test_ctypes_binding_matches_the_header(lib):
    header = open(os.path.join(ROOT, "include", "nsb.h")).read()
    m = re.search(r"int nsb_render_forward_interp\(([^)]*)\);", header)
    assert m, "nsb_render_forward_interp is declared in nsb.h"
    params = [re.sub(r"/\*.*?\*/", "", x).split()[-2:] for x in m.group(1).split(",")]
    assert [" ".join(p) for p in params] == ["nsb_field_params *params", "nsb_field_opts *opts", "nsb_render_args *args",
                                             "void *stream"], params
    fn = lib.nsb_render_forward_interp
    assert fn.restype is C.c_int
    assert list(fn.argtypes) == [C.POINTER(_lib.FieldParams), C.POINTER(_lib.FieldOpts), C.POINTER(_lib.RenderArgs), C.c_void_p]
    assert list(fn.argtypes) == list(lib.nsb_render_forward.argtypes)


def test_linear_kernels_compile_for_sm90a_within_the_spill_budget():
    """The four render_kernel_tc_lerp instantiations: tensor-role spills within the wgmma kernels' budget and gather-role
    spills no more than the nearest kernel of the same shape, counted with the region rule of test_tc_spill_cpu."""
    import test_tc_spill_cpu as sp
    if not os.path.exists(sp.OBJ):
        pytest.skip("needs the in-tree object (make -C nersemble_b200/csrc)")
    rows = sp._region_spills(sp.OBJ)
    for sampler in (2, 4):
        for shape in ("Lb1ELb1E", "Lb0ELb0E"):
            lerp = [k for k in rows if f"render_kernel_tc_lerpILi{sampler}E{shape}" in k]
            near = [k for k in rows if f"render_kernel_tcILi{sampler}E{shape}" in k]
            assert len(lerp) == 1 and len(near) == 1, (lerp, near)
            r, n = rows[lerp[0]], rows[near[0]]
            assert r["pre"] == 0 and r["tensor"] <= sp.TENSOR_MAX and r["gather"] <= n["gather"], (lerp[0], r, n)
