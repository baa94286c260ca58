"""CPU tests of the mesh export: the numpy oracle on closed surfaces (watertight, consistently wound, right topology and
volume), the kernel's documented winding rule against the oracle's geometric one, the host-side checks of the two entry
points, a compile-and-spill guard for nsb_mesh.cu, the ctypes mirror of nsb_mesh_args, the grid rule of mesh_grid and the
PLY round trip."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import mesh_oracle as mo
from conftest import ROOT

CSRC = os.path.join(ROOT, "nersemble_b200", "csrc")
DUMMY = 0x10000      # non-null, never dereferenced: every call below is rejected on the host


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_oracle_mesh_is_closed_and_oriented(shape):
    """Every undirected edge is in exactly two faces, once in each direction; V - E + F is 2 for the sphere and 0 for
    the torus; the signed volume is positive and within 2 % of the analytic one."""
    if shape == "sphere":
        fn, vol, chi = mo.sphere(0.7), 4.0 / 3.0 * math.pi * 0.7 ** 3, 2
    else:
        fn, vol, chi = mo.torus(0.55, 0.25), 2.0 * math.pi ** 2 * 0.55 * 0.25 ** 2, 0
    sigma, box_min, h = mo.sample_grid(fn, 41)
    v, f = mo.marching_tetrahedra(sigma, 0.0, box_min, h)
    assert len(f) > 1000
    edges, uses, n_fwd = mo.edge_use(f)
    assert (uses == 2).all() and (n_fwd == 1).all()
    assert len(v) - len(edges) + len(f) == chi
    got = mo.signed_volume(v, f)
    assert got > 0 and abs(got / vol - 1.0) < 0.02, (got, vol)
    # every vertex is used, and lies on the surface's grid edge
    assert np.array_equal(np.unique(f), np.arange(len(v)))


def test_oracle_order_on_a_small_grid():
    """Vertex ids follow (grid point, slot); faces follow (cell, tetrahedron, triangle).  One inside point in a 3^3 grid:
    its 7 owned edges cross plus the edges of the lower neighbours that end at it."""
    sigma = np.zeros((3, 3, 3), np.float32)
    sigma[1, 1, 1] = 2.0
    v, f = mo.marching_tetrahedra(sigma, 1.0, [0.0] * 3, [1.0] * 3)
    # the first vertex belongs to point 0 (slot +x+y+z reaches (1,1,1)), at the edge's midpoint
    assert np.allclose(v[0], [0.5, 0.5, 0.5])
    assert mo.signed_volume(v, f) > 0
    edges, uses, n_fwd = mo.edge_use(f)
    assert (uses == 2).all() and (n_fwd == 1).all()


def _parity_rule(t, pattern):
    """The kernel's winding rule (nsb_mesh.cu, DESIGN 4.2d) written out: parity P of tetrahedron t, corners 0..3."""
    P = [1, -1, -1, 1, 1, -1][t]
    ins = [c for c in range(4) if (pattern >> c) & 1]
    outs = [c for c in range(4) if not (pattern >> c) & 1]
    if len(ins) in (1, 3):
        lone = ins[0] if len(ins) == 1 else outs[0]
        rest = outs if len(ins) == 1 else ins
        sgn = (-1) ** lone * P * (1 if len(ins) == 1 else -1)
        a, b, c = [(lone, r) for r in rest]
        return [[a, b, c] if sgn > 0 else [a, c, b]]
    if len(ins) == 2:
        (i, j), (k, l) = ins, outs
        if (-1) ** (i + j + 1) * P > 0:
            return [[(i, k), (i, l), (j, l)], [(i, k), (j, l), (j, k)]]
        return [[(i, k), (j, k), (j, l)], [(i, k), (j, l), (i, l)]]
    return []


def test_kernel_winding_rule_matches_the_geometric_orientation():
    table = mo.case_table()
    for t in range(6):
        for pattern in range(16):
            assert _parity_rule(t, pattern) == table[t][pattern], (t, pattern)


def test_tetrahedron_parity_is_the_orientation():
    for t, corners in enumerate(mo.tetrahedra()):
        det = round(np.linalg.det(np.stack([corners[1] - corners[0], corners[2] - corners[0], corners[3] - corners[0]])))
        assert det == [1, -1, -1, 1, 1, -1][t]


# ------------------------------------------------------------------ entry points
@pytest.fixture(scope="module")
def lib():
    from nersemble_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib.load()


def _args():
    from nersemble_b200 import _lib
    a = _lib.MeshArgs()
    a.sigma = a.point_mask = a.vertex_base = a.tile_sums = a.vertices = a.faces = DUMMY
    a.nx, a.ny, a.nz, a.level = 8, 8, 8, 0.5
    a.n_vertices, a.n_faces = 10, 10
    return a


def _flat(a):
    a.nx = 1


def _huge(a):
    a.nx, a.ny, a.nz = 2048, 1024, 1024


def _nan_level(a):
    a.level = float("nan")


def _inf_level(a):
    a.level = float("inf")


def _no_sigma(a):
    a.sigma = None


def _no_mask(a):
    a.point_mask = None


CASES = [("nx = 1", _flat, "every grid dimension must be >= 2"),
         ("2^31 points", _huge, "the grid must have fewer than 2^31 points"),
         ("nan level", _nan_level, "level must be finite"),
         ("inf level", _inf_level, "level must be finite"),
         ("no sigma", _no_sigma, "sigma, point_mask and tile_sums are required"),
         ("no point_mask", _no_mask, "sigma, point_mask and tile_sums are required")]


@pytest.mark.parametrize("entry", ["nsb_mesh_count", "nsb_mesh_emit"])
@pytest.mark.parametrize("case,breaks,message", CASES, ids=[c[0] for c in CASES])
def test_mesh_entry_points_reject_on_the_host(lib, entry, case, breaks, message):
    a = _args()
    breaks(a)
    rc = getattr(lib, entry)(C.byref(a), None)
    err = lib.nsb_last_error().decode()
    assert rc != 0 and err == f"{entry}: {message}", err


@pytest.mark.parametrize("field,value,message", [
    ("n_vertices", 1 << 31, "n_vertices and n_faces must be in [0, 2^31)"),
    ("n_faces", 1 << 31, "n_vertices and n_faces must be in [0, 2^31)"),
    ("n_faces", -1, "n_vertices and n_faces must be in [0, 2^31)"),
    ("vertices", None, "vertex_base, vertices and faces are required"),
    ("faces", None, "vertex_base, vertices and faces are required"),
    ("vertex_base", None, "vertex_base, vertices and faces are required")])
def test_mesh_emit_rejects_its_outputs_on_the_host(lib, field, value, message):
    a = _args()
    setattr(a, field, value)
    rc = lib.nsb_mesh_emit(C.byref(a), None)
    err = lib.nsb_last_error().decode()
    assert rc != 0 and err == f"nsb_mesh_emit: {message}", err


def test_mesh_args_mirror_matches_the_c_header(tmp_path):
    from nersemble_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nsb.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(nsb_mesh_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(nsb_mesh_args, {f}));' for f, _ in _lib.MeshArgs._fields_]
    lines += ['  printf("tile %d\\n", NSB_MESH_TILE);', '  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got.pop("size")) == C.sizeof(_lib.MeshArgs)
    assert int(got.pop("tile")) == _lib.MESH_TILE
    for f, _ in _lib.MeshArgs._fields_:
        assert int(got[f]) == getattr(_lib.MeshArgs, f).offset, f


def test_mesh_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("needs nvcc")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", os.path.join(CSRC, "nsb_mesh.cu"),
                          "-o", str(tmp_path / "nsb_mesh.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "warning" not in out.stderr.lower(), out.stderr
    blocks = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                        out.stderr)
    kernels = {b[0] for b in blocks if "mesh_" in b[0]}
    assert len(kernels) == 4, out.stderr
    for name, stack, st, ld in blocks:
        assert int(stack) == 0 and int(st) == 0 and int(ld) == 0, (name, stack, st, ld)


# ------------------------------------------------------------------ host side of the op and the export
def test_mesh_grid_rule():
    from nersemble_b200 import ops

    class P:
        aabb_list = [-2.5, -1.8, -2.5, 2.2, 1.8, 2.0]
    box_min, h, dims = ops.mesh_grid(P, 256)
    assert dims[0] == 256 and h[0] == h[1] == h[2] and h[0] == float(np.float32(4.7 / 255))
    for k in range(3):     # the grid ends within half a voxel of the box
        end = box_min[k] + (dims[k] - 1) * h[k]
        assert abs(end - P.aabb_list[3 + k]) <= 0.5 * h[k] + 1e-6
    box_min, h, dims = ops.mesh_grid(P, (64, 48, 40), box=[[0, 0, 0], [1, 2, 3]])
    assert dims == (64, 48, 40) and box_min == [0.0, 0.0, 0.0]
    assert h == [float(np.float32(1 / 63)), float(np.float32(2 / 47)), float(np.float32(3 / 39))]
    with pytest.raises(ValueError):
        ops.mesh_grid(P, 1)
    with pytest.raises(ValueError):
        ops.mesh_grid(P, (4, 4))


def test_ply_round_trip(tmp_path):
    from nersemble_b200.mesh import Mesh
    sigma, box_min, h = mo.sample_grid(mo.sphere(0.6), 17)
    v, f = mo.marching_tetrahedra(sigma, 0.0, box_min, h)
    rng = np.random.default_rng(0)
    nrm = rng.standard_normal(v.shape).astype(np.float32)
    rgb = rng.random(v.shape).astype(np.float32)
    for normals, colours in ((nrm, rgb), (None, None), (nrm, None)):
        m = Mesh(v, f, normals, colours)
        path = str(tmp_path / "m.ply")
        m.save_ply(path)
        with open(path, "rb") as fh:
            assert fh.read(3) == b"ply"
        back = Mesh.load_ply(path)
        assert np.array_equal(back.vertices, v) and np.array_equal(back.faces, f)
        assert (back.normals is None) == (normals is None) and (back.colours is None) == (colours is None)
        if normals is not None:
            assert np.array_equal(back.normals, nrm)
        if colours is not None:
            assert np.abs(back.colours - rgb).max() <= 0.5 / 255 + 1e-7
    empty = Mesh(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    empty.save_ply(str(tmp_path / "e.ply"))
    back = Mesh.load_ply(str(tmp_path / "e.ply"))
    assert back.vertices.shape == (0, 3) and back.faces.shape == (0, 3)
