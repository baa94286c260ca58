"""Surface normals without a GPU: the oracle's autograd normals against central finite differences of its own h0, the
ctypes mirror of nsb_normals_args against the C header, and the normals kernel's SASS (no local-memory traffic)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from conftest import ROOT
from normals_oracle import field_normals, h0
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision


def test_oracle_normals_match_finite_differences():
    """At points where no level changes cell and no ReLU switches within +-eps (h0 is smooth there), the autograd
    gradient is the central difference of h0.  fp32 math without fp16 activations ("none"), so h0 is exactly piecewise multilinear in x."""
    Precision.mode = "none"
    try:
        P = pl.random_params(n_timesteps=2, log2_hashmap_size=12, table_scale=1.0)
        gen = torch.Generator().manual_seed(5)
        n, eps = 400, 1e-6
        # near the box origin: the oracle rounds pos = scale * x + 0.5 to float32, a quantisation that grows with x
        x = 0.01 + 0.09 * torch.rand((n, 3), generator=gen)
        codes = torch.randn((n, 32), generator=gen) * 0.3
        pos = P.aabb[0] + x * (P.aabb[1] - P.aabb[0])
        _, g = field_normals(P, pos, codes, None)
        xs = (pos - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
        lv = P.levels
        fd = torch.zeros_like(g)
        same = torch.ones(n, dtype=torch.bool)
        for k in range(3):
            e = torch.zeros(3); e[k] = eps
            xp, xm = xs + e, xs - e
            for l in range(lv.n_levels):
                s = float(lv.scale[l])
                same &= ((xp[:, k].double() * s + 0.5).float().floor() == (xm[:, k].double() * s + 0.5).float().floor())
            with torch.no_grad():
                fd[:, k] = (h0(P, xp, codes, None) - h0(P, xm, codes, None)) / (xp[:, k] - xm[:, k])
                # ... and no hidden ReLU of mlp_base switches within the step
                hid = [pl.hash_ensemble(P, xx, codes, None) @ P.base_w[0].half().float().t() > 0 for xx in (xp, xm)]
                same &= (hid[0] == hid[1]).all(-1)
        assert same.sum() > 200, same.sum()
        err = (fd - g)[same].norm(dim=-1) / g[same].norm(dim=-1)
        assert err.median() < 2e-3 and err.max() < 1e-2, (err.median(), err.max())
        # the normal of a sample outside the box is the gradient at the box origin (x = 0), not zero
        n_out, g_out = field_normals(P, P.aabb[1][None] + 1.0, codes[:1], None)
        n_org, g_org = field_normals(P, P.aabb[0][None], codes[:1], None)
        assert g_out.norm() > 0 and torch.equal(g_out, g_org)
    finally:
        Precision.mode = "reference"


def test_normals_args_ctypes_layout_matches_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc")
    from nersemble_b200 import _lib
    cls = _lib.NormalsArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nsb.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(nsb_normals_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(nsb_normals_args, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = {a: int(b) for a, b in (l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                     check=True).stdout.splitlines())}
    want = {"size": ctypes.sizeof(cls), **{f: getattr(cls, f).offset for f, _ in cls._fields_}}
    assert got == want


def test_normals_kernels_have_no_local_memory_traffic():
    obj = os.path.join(ROOT, "nersemble_b200", "csrc", "nsb_normals.o")
    if not os.path.exists(obj) or shutil.which("cuobjdump") is None:
        pytest.skip("needs the in-tree object file and cuobjdump")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels = re.split(r"\n\s*Function : ", sass)[1:]
    names = [k.split("\n", 1)[0] for k in kernels]
    assert sum("normals_kernel" in n for n in names) == 2 and any("normals_composite_kernel" in n for n in names), names
    for name, body in zip(names, kernels):
        assert not re.search(r"\b(STL|LDL)\b", body), name
