"""The deformation's Jacobian and inverse without a GPU: the float64 Newton oracle against the analytic inverse of a rigid
warp, the forward-mode oracle J against the pullback oracle J, the ctypes mirrors of the new argument structs, the
host-side checks of nsb_deform_jacobian / nsb_deform_inverse, a spill-free sm_90a compile, and the MeshSequence PLY round
trip."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from deform_inverse_oracle import (as_float64, jacobian_by_pullbacks, jacobian_jacfwd, newton_inverse, rigid_inverse,
                                   rigid_params)
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision


@pytest.fixture
def no_rounding():
    old = Precision.mode
    Precision.mode = "none"
    yield
    Precision.mode = old


@pytest.mark.parametrize("r", [(0.1, -0.15, 0.12), (3e-3, -2e-3, 1e-3)], ids=["rotation", "clamped_theta"])
def test_float64_newton_oracle_inverts_a_rigid_warp(no_rounding, r):
    P = rigid_params(r, (0.02, -0.03, 0.01))
    P64 = as_float64(P)
    gen = torch.Generator().manual_seed(0)
    c = 0.3 + 0.4 * torch.rand((200, 3), generator=gen, dtype=torch.float64)
    pos, res = newton_inverse(P64, c, torch.zeros((200, 128)), 7.0)
    assert res.max() < 1e-13
    assert (pos - rigid_inverse(c, P64.r_b, P64.v_b)).abs().max().item() <= 1e-12


def test_forward_mode_jacobian_equals_the_pullback_oracle():
    """torch.func.jacfwd through the oracle's warp equals the three pullbacks of deform_jacobian_oracle, with and without
    the posenc window."""
    P = pl.random_params(n_timesteps=3, log2_hashmap_size=4, deform_last_scale=2e-2)
    gen = torch.Generator().manual_seed(2)
    n = 200
    pn = torch.rand((n, 3), generator=gen)
    wc = P.time_emb_deform[torch.randint(0, 3, (n,), generator=gen)] * 100.0
    pos = P.aabb[0] + pn * (P.aabb[1] - P.aabb[0])
    pn = (pos - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    for window in (None, 3.5):
        a = jacobian_jacfwd(P, pn, wc, window)
        b = jacobian_by_pullbacks(P, pos, wc, window)
        assert b.norm(dim=(-2, -1)).median() > 1e-2
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("struct,ctype", [("nsb_deform_jac_args", "DeformJacArgs"), ("nsb_deform_inv_args", "DeformInvArgs")])
def test_ctypes_layout_matches_the_header(tmp_path, struct, ctype):
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc")
    from nersemble_b200 import _lib
    cls = getattr(_lib, ctype)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nsb.h"', 'int main(void) {',
             f'  printf("size %zu\\n", sizeof({struct}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({struct}, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = {a: int(b) for a, b in (l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                     check=True).stdout.splitlines())}
    assert got == {"size": ctypes.sizeof(cls), **{f: getattr(cls, f).offset for f, _ in cls._fields_}}


def _lib_loaded():
    from nersemble_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib.load()


def _positions_samples():
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    s = _lib.Samples()
    s.n_samples = 256
    s.positions = s.sample_times = ec.DUMMY
    return s


def _jac(lib, p, s, a=None):
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    if a is None:
        a = ec._fill(_lib.DeformJacArgs())
        a.tangent_scale = 1.0 / 16
    return lib.nsb_deform_jacobian(ctypes.byref(p), ctypes.byref(ec._opts()), ctypes.byref(s), ctypes.byref(a), None)


def _inv(lib, p, s, a=None):
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    if a is None:
        a = _inv_args()
    return lib.nsb_deform_inverse(ctypes.byref(p), ctypes.byref(ec._opts()), ctypes.byref(s), ctypes.byref(a), None)


def _inv_args(**over):
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    a = ec._fill(_lib.DeformInvArgs(), skip=("init",))
    a.tangent_scale, a.max_iter, a.tol = 1.0 / 16, 20, 1e-4
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("entry", ["nsb_deform_jacobian", "nsb_deform_inverse"])
def test_entry_points_reject_bad_inputs_on_the_host(entry):
    """Every check runs before any CUDA call and names the entry point; the pointers are never dereferenced."""
    import test_entry_checks_cpu as ec
    lib = _lib_loaded()
    call = _jac if entry == "nsb_deform_jacobian" else _inv

    def expect(rc, message):
        err = lib.nsb_last_error().decode()
        assert rc != 0 and err == f"{entry}: {message}", err

    for _, breaks, message in ec.CASES[:2]:          # the field-parameter checks every field entry point runs
        p, s = ec._params(), _positions_samples()
        breaks(p, s)
        expect(call(lib, p, s), message)
    p = ec._params()
    expect(call(lib, p, ec._samples()), "positions-based samples only")
    s = _positions_samples(); s.positions = None
    expect(call(lib, p, s), "no sample source")
    p.deform_packed_tb = None
    expect(call(lib, p, _positions_samples()), "missing deformation parameters")
    p = ec._params(); p.deform_code_bias = None
    expect(call(lib, p, _positions_samples()), "missing deformation parameters")
    p = ec._params()
    if entry == "nsb_deform_jacobian":
        from nersemble_b200 import _lib
        a = ec._fill(_lib.DeformJacArgs(), skip=("jacobian",)); a.tangent_scale = 1.0 / 16
        expect(_jac(lib, p, _positions_samples(), a), "null output")
        a = ec._fill(_lib.DeformJacArgs()); a.tangent_scale = 0.0
        expect(_jac(lib, p, _positions_samples(), a), "tangent_scale must be finite and > 0")
    else:
        for mi in (0, 65, -3):
            expect(_inv(lib, p, _positions_samples(), _inv_args(max_iter=mi)), f"max_iter must be in 1..64, got {mi}")
        for tol in (0.0, -1e-4, float("nan"), float("inf")):
            expect(_inv(lib, p, _positions_samples(), _inv_args(tol=tol)), "tol must be finite and > 0")
        for out in ("positions", "residual", "iterations", "status"):
            expect(_inv(lib, p, _positions_samples(), _inv_args(**{out: None})), "null output")
        expect(_inv(lib, p, _positions_samples(), _inv_args(tangent_scale=float("inf"))),
               "tangent_scale must be finite and > 0")


def test_python_arguments_are_validated_before_any_device_call():
    from nersemble_b200 import ops
    pos = torch.zeros((4, 3))
    for mi in (0, 65, 2.5):
        with pytest.raises(ValueError, match="max_iter"):
            ops.deform_inverse(None, pos, max_iter=mi)
    for tol in (0.0, float("nan")):
        with pytest.raises(ValueError, match="tol"):
            ops.deform_inverse(None, pos, tol=tol)
    with pytest.raises(ValueError, match="positions-based"):
        ops.deform_jacobian(None, origins=pos, directions=pos, t_starts=pos[:, 0], t_ends=pos[:, 0],
                            ray_indices=torch.zeros(4, dtype=torch.int32))
    with pytest.raises(ValueError, match="one of"):
        ops.deform_inverse(None, pos, sample_times=torch.zeros(4), uniform_time=0.5)


def test_deform_inv_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("needs nvcc")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                          os.path.join(ROOT, "nersemble_b200", "csrc", "nsb_deform_inv.cu"),
                          "-o", str(tmp_path / "nsb_deform_inv.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "warning" not in out.stderr.lower(), out.stderr
    blocks = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                        r"\s+ptxas info\s+: Used (\d+) registers", out.stderr)
    kernels = [b for b in blocks if "deform_inv_kernel" in b[0]]
    assert len(kernels) == 2, out.stderr
    for _, stack, st, ld, regs in kernels:
        # sinf / sincosf keep their 32-byte argument-reduction table on the stack; that is not a spill
        assert int(st) == 0 and int(ld) == 0 and int(stack) <= 64 and int(regs) <= 255, kernels
    from nersemble_b200 import _lib
    for name in ("nsb_deform_jacobian", "nsb_deform_inverse"):
        assert hasattr(_lib_loaded(), name)


def test_mesh_sequence_ply_round_trip(tmp_path):
    from nersemble_b200.mesh import Mesh, MeshSequence
    rng = np.random.default_rng(0)
    K, V, F = 3, 50, 80
    seq = MeshSequence(faces=rng.integers(0, V, (F, 3)).astype(np.int32),
                       vertices=rng.standard_normal((K, V, 3)).astype(np.float32), timesteps=[4, 7, 9],
                       converged=rng.random((K, V)) > 0.1, sigma=rng.random((K, V)).astype(np.float32),
                       normals=rng.standard_normal((K, V, 3)).astype(np.float32), colours=rng.random((K, V, 3)).astype(np.float32))
    assert len(seq) == 3
    paths = seq.save_ply(str(tmp_path / "f{:03d}.ply"))
    assert [os.path.basename(p) for p in paths] == ["f004.ply", "f007.ply", "f009.ply"]
    for i, p in enumerate(paths):
        back = Mesh.load_ply(p)
        fr = seq.frame(i)
        assert np.array_equal(back.vertices, seq.vertices[i]) and np.array_equal(back.faces, seq.faces)
        assert np.array_equal(back.normals, fr.normals)
        assert np.abs(back.colours - fr.colours).max() <= 0.5 / 255 + 1e-7
    with pytest.raises(ValueError, match="same file"):
        seq.save_ply(str(tmp_path / "same.ply"))
    bare = MeshSequence(seq.faces, seq.vertices, seq.timesteps, seq.converged, seq.sigma)
    assert bare.frame(1).normals is None and bare.frame(1).colours is None
