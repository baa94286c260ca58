"""The flow pass without a GPU: pi against the ray generation, the oracle's per-ray sums on hand-made packed samples, the
ctypes mirrors of the new argument structs, the host-side checks of nsb_flow_select / nsb_flow_composite, the Python
argument checks of ops.render_flow and a spill-free sm_90a compile."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

from conftest import ROOT
from flow_oracle import composite, project, ray_directions, select

INTR = (800.0, 790.0, 40.3, 29.6)


def _c2w():
    """A camera 9 units from the origin looking at it (-z forward, +y up), as in test_gpu_rays.py."""
    eye = torch.tensor([9 * math.sin(0.7), 0.4, 9 * math.cos(0.7)], dtype=torch.float64)
    fwd = -eye / eye.norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64)); right = right / right.norm()
    up = torch.linalg.cross(right, fwd)
    return torch.cat([torch.stack([right, up, -fwd], -1), eye[:, None]], -1)


def test_projection_inverts_the_ray_generation():
    c2w = _c2w()
    rows, cols = torch.meshgrid(torch.arange(0, 60, 7), torch.arange(0, 80, 9), indexing="ij")
    rows, cols = rows.reshape(-1), cols.reshape(-1)
    d = ray_directions(INTR, c2w, rows, cols)
    for t in (0.5, 9.0, 37.0):
        pix, front = project(c2w[:, 3] + t * d, INTR, c2w)
        assert front.all()
        want = torch.stack([cols.double() + 0.5, rows.double() + 0.5], -1)
        assert (pix - want).abs().max().item() <= 1e-9
    _, front = project(c2w[:, 3] - 2.0 * d, INTR, c2w)
    assert not front.any()


def _packed():
    """4 rays: ray 0 empty, ray 1 with all weights below min_weight (W = 0), ray 2 with a non-converged sample and one
    exactly at min_weight, ray 3 with samples past n_total (garbage slots)."""
    mw = 1e-3
    info = torch.tensor([[0, 0], [0, 3], [3, 4], [7, 3]])
    w = torch.tensor([1e-4, 5e-4, 9.99e-4, 0.5, mw, 2e-4, 0.25, 0.3, float("nan"), 0.9])
    n = w.shape[0]
    g = torch.Generator().manual_seed(0)
    ts = torch.rand(n, generator=g) * 4 + 5
    te = ts + 0.01
    off = torch.randn((n, 3), generator=g) * 0.01
    o = torch.randn((4, 3), generator=g)
    d = torch.nn.functional.normalize(torch.randn((4, 3), generator=g), dim=-1)
    return info, ts, te, w, off, o, d, mw


def test_oracle_selection_and_per_ray_sums_on_hand_made_samples():
    info, ts, te, w, off, o, d, mw = _packed()
    s = select(info, ts, te, w, off, o, d, n_total=8, min_weight=mw)
    assert s["sel_index"].tolist() == [3, 4, 6, 7]          # 4 is exactly at min_weight; 8, 9 are past n_total
    assert s["ray_sel"].tolist() == [[0, 0], [0, 0], [0, 3], [3, 1]] and s["n_selected"] == 4
    x = o[2] + (d[2] * (ts[3] + te[3])) * 0.5
    assert torch.equal(s["init"][0], x) and torch.equal(s["targets"][0], x + off[3])
    moved = s["init"].double() + torch.tensor([[0.1, 0.0, 0.0], [0.0, 0.2, 0.0], [0.0, 0.0, 0.3], [0.05, 0.05, 0.05]],
                                              dtype=torch.float64)
    status = torch.tensor([0, 0, 1, 0], dtype=torch.int32)                  # sample 6 did not converge
    out = composite(s["ray_sel"], s["sel_index"], s["init"], moved, status, w)
    W, w64 = out["flow_weight"], w.double()
    assert W[0] == 0 and W[1] == 0 and W[2] == w64[3] + w64[4] and W[3] == w64[7]
    want2 = (w64[3] * torch.tensor([0.1, 0.0, 0.0], dtype=torch.float64)
             + w64[4] * torch.tensor([0.0, 0.2, 0.0], dtype=torch.float64)) / (w64[3] + w64[4])
    assert (out["scene_flow"][2] - want2).abs().max() < 1e-12
    assert (out["scene_flow"][3] - 0.05).abs().max() < 1e-12
    assert (out["scene_flow"][:2] == 0).all()
    # a camera: sample 7 behind it is left out of the optical flow only
    c2w = _c2w()
    cam_x = c2w[:, 3] - 3.0 * c2w[:, 2]                # 3 units in front of the camera
    init = s["init"].double().clone(); init[:3] = cam_x
    init[3] = c2w[:, 3] + 3.0 * c2w[:, 2]              # behind
    moved = init + torch.tensor([[0.01, 0.0, 0.0]] * 4, dtype=torch.float64)
    out = composite(s["ray_sel"], s["sel_index"], init, moved, status, w, camera=(INTR, c2w))
    p0, _ = project(init[:1], INTR, c2w)
    p1, _ = project(moved[:1], INTR, c2w)
    assert (out["optical_flow"][2] - (p1 - p0)[0]).abs().max() < 1e-9
    assert (out["optical_flow"][3] == 0).all() and out["flow_weight"][3] == w64[7]
    assert (out["optical_flow"][:2] == 0).all()


@pytest.mark.parametrize("struct,ctype", [("nsb_flow_select_args", "FlowSelectArgs"),
                                          ("nsb_flow_composite_args", "FlowCompositeArgs")])
def test_ctypes_layout_matches_the_header(tmp_path, struct, ctype):
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc")
    from nersemble_b200 import _lib
    cls = getattr(_lib, ctype)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nsb.h"', 'int main(void) {',
             f'  printf("size %zu\\n", sizeof({struct}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({struct}, {f}));' for f, _ in cls._fields_]
    lines += [f'  printf("tile %d\\n", NSB_FLOW_TILE);', '  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = {a: int(b) for a, b in (l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                     check=True).stdout.splitlines())}
    assert got == {"size": ctypes.sizeof(cls), "tile": _lib.FLOW_TILE, **{f: getattr(cls, f).offset for f, _ in cls._fields_}}


def _lib_loaded():
    from nersemble_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib.load()


def _select_args(**over):
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    a = ec._fill(_lib.FlowSelectArgs())
    a.n_rays, a.capacity, a.min_weight = 16, 256, 1e-3
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _composite_args(camera=True, **over):
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    a = ec._fill(_lib.FlowCompositeArgs(), skip=() if camera else ("optical_flow",))
    a.n_rays, a.capacity = 16, 256
    a.intrinsics[:] = INTR
    a.camera_to_world[:] = [float(v) for v in _c2w().reshape(-1)]
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_entry_points_reject_bad_inputs_on_the_host():
    """Every check runs before any CUDA call and names the entry point; the pointers are never dereferenced."""
    lib = _lib_loaded()

    def expect(entry, a, message):
        fn = getattr(lib, entry)
        rc = fn(None if a is None else ctypes.byref(a), None)
        err = lib.nsb_last_error().decode()
        assert rc != 0 and err == f"{entry}: {message}", err

    expect("nsb_flow_select", None, "null argument")
    expect("nsb_flow_composite", None, "null argument")
    for entry, make in (("nsb_flow_select", _select_args), ("nsb_flow_composite", _composite_args)):
        expect(entry, make(n_rays=-1), "n_rays must be >= 0")
        for cap in (0, -5):
            expect(entry, make(capacity=cap), "capacity must be > 0")
        for name, _ in make()._fields_:
            if name in ("n_rays", "capacity", "min_weight", "intrinsics", "camera_to_world", "optical_flow"):
                continue
            expect(entry, make(**{name: None}), "null pointer")
    for mw in (-1e-3, 1.0, 2.0, float("nan"), float("inf")):
        expect("nsb_flow_select", _select_args(min_weight=mw), "min_weight must be finite and in [0, 1)")
    for k in range(4):
        a = _composite_args(); a.intrinsics[k] = float("nan")
        expect("nsb_flow_composite", a, "camera values must be finite")
    for k in (0, 5, 11):
        a = _composite_args(); a.camera_to_world[k] = float("inf")
        expect("nsb_flow_composite", a, "camera values must be finite")
    for k, v in ((0, 0.0), (1, -790.0)):
        a = _composite_args(); a.intrinsics[k] = v
        expect("nsb_flow_composite", a, "fx and fy must be > 0")
    # without a camera its values are not read
    a = _composite_args(camera=False, n_rays=0); a.intrinsics[0] = float("nan")
    assert lib.nsb_flow_composite(ctypes.byref(a), None) == 0


def test_python_arguments_are_validated_before_any_device_call():
    from nersemble_b200 import ops
    for t in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="time_to"):
            ops.render_flow(None, None, None, None, None, time_to=t)
    for mw in (-1e-3, 1.0, float("nan")):
        with pytest.raises(ValueError, match="min_weight"):
            ops.render_flow(None, None, None, None, None, time_to=0.5, min_weight=mw)
    for mi in (0, 65, 2.5):
        with pytest.raises(ValueError, match="max_iter"):
            ops.render_flow(None, None, None, None, None, time_to=0.5, max_iter=mi)
    with pytest.raises(ValueError, match="tol"):
        ops.render_flow(None, None, None, None, None, time_to=0.5, tol=0.0)
    c2w = _c2w()
    bad = [((1.0, 2.0, 3.0), c2w, "camera must be"), (INTR, c2w[:, :3], "camera must be"),
           ((float("nan"), 1.0, 2.0, 3.0), c2w, "finite"), ((0.0, 1.0, 2.0, 3.0), c2w, "fx and fy")]
    for intr, c, match in bad:
        with pytest.raises(ValueError, match=match):
            ops.render_flow(None, None, None, None, None, time_to=0.5, camera=(intr, c))
    with pytest.raises(ValueError, match="camera must be"):
        ops.render_flow(None, None, None, None, None, time_to=0.5, camera=INTR)


def test_flow_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("needs nvcc")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                          os.path.join(ROOT, "nersemble_b200", "csrc", "nsb_flow.cu"),
                          "-o", str(tmp_path / "nsb_flow.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "warning" not in out.stderr.lower(), out.stderr
    blocks = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                        r"\s+ptxas info\s+: Used (\d+) registers", out.stderr)
    kernels = [b for b in blocks if "flow_" in b[0]]
    assert len(kernels) == 4, out.stderr
    for _, stack, st, ld, regs in kernels:
        assert int(st) == 0 and int(ld) == 0 and int(stack) == 0 and int(regs) <= 255, kernels
    for name in ("nsb_flow_select", "nsb_flow_composite"):
        assert hasattr(_lib_loaded(), name)
