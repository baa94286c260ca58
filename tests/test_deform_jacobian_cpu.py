"""The deformation's input Jacobian without a GPU: the autograd oracle against float64 finite differences of the oracle's
own offsets, the packer of the transposed posenc block against a plain matrix product, the ctypes mirror of
nsb_deform_vjp_args, the host-side checks of nsb_deform_input_grad, and argument validation before any device call."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from conftest import ROOT
from deform_jacobian_oracle import offsets_of_normalised, offsets_vjp
from oracle import pipeline as pl


def test_oracle_vjp_matches_float64_finite_differences():
    """reference precision (no fp16 rounding): central differences of the oracle's float32 offsets, the quotient formed
    in float64.  The step follows the highest band the window lets through (h = 1e-3 at 1.5, 3e-4 at 3.5, 3e-5 with all
    seven bands: 2 pi 64), where truncation and float32 noise over 2 h balance: the median row agrees to 2e-3
    (measured), the tail are rows where a stem ReLU switches within the step."""
    P = pl.random_params(n_timesteps=3, log2_hashmap_size=4, deform_last_scale=2e-2)
    gen = torch.Generator().manual_seed(2)
    n = 400
    pn = torch.rand((n, 3), generator=gen)
    wc = P.time_emb_deform[torch.randint(0, 3, (n,), generator=gen)] * 100.0
    u = torch.randn((n, 3), generator=gen)
    pos = P.aabb[0] + pn * (P.aabb[1] - P.aabb[0])
    pn_r = (pos - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    for window, h in ((1.5, 1e-3), (3.5, 3e-4), (None, 3e-5)):
        got = offsets_vjp(P, pos, wc, window, u).double()
        fd = torch.zeros((n, 3), dtype=torch.float64)
        with torch.no_grad():
            for k in range(3):
                e = torch.zeros(3); e[k] = h
                xp, xm = pn_r + e, pn_r - e
                diff = offsets_of_normalised(P, xp, wc, window).double() - offsets_of_normalised(P, xm, wc, window).double()
                fd[:, k] = (diff * u.double()).sum(-1) / (xp[:, k].double() - xm[:, k].double())
        rel = (got - fd).norm(dim=-1) / fd.norm(dim=-1)
        assert fd.norm(dim=-1).median() > 1e-2           # not the ~1e-5 of freshly initialised heads
        assert rel.median() < 5e-3 and (rel < 0.2).float().mean() > 0.95, (window, rel.median(), rel.max())


def test_posenc_block_packer_is_the_transposed_matrix_product():
    """delta [16 x 128] times the packed block, multiplied out the way mma.sync m16n8k16 reads B fragments, equals
    delta @ W[:, posenc columns in kernel order] (padding columns zero) for layers 0 and 4."""
    from nersemble_b200 import packing
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn((128, 173), generator=gen)
    w4 = torch.randn((128, 301), generator=gen)
    packed = packing.pack_deform_pe_t(w0, w4)
    assert packed.dtype == torch.float16 and packed.numel() == 2 * 8 * 3 * 32 * 8
    cm = packing.deform_input_colmap()[:48]
    delta = torch.randn((16, 128), generator=gen).half().float()
    for blk, w in enumerate((w0, w4)):
        frag = packed[blk * 6144:(blk + 1) * 6144].float().view(8, 3, 8, 4, 2, 2, 2)     # kt, pair, g, q, ntsel, hi, e
        B = torch.zeros((128, 48))                                                       # [k][n]
        for kt in range(8):
            for pair in range(3):
                for g in range(8):
                    for q in range(4):
                        for ntsel in range(2):
                            for hi in range(2):
                                for e in range(2):
                                    B[kt * 16 + hi * 8 + 2 * q + e, pair * 16 + ntsel * 8 + g] = frag[kt, pair, g, q, ntsel, hi, e]
        want = torch.stack([w[:, c].half().float() if c >= 0 else torch.zeros(128) for c in cm], 1)   # [128, 48]
        assert torch.equal(B, want)
        torch.testing.assert_close(delta @ B, delta @ want)


def test_deform_vjp_args_ctypes_layout_matches_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc")
    from nersemble_b200 import _lib
    cls = _lib.DeformVjpArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nsb.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(nsb_deform_vjp_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(nsb_deform_vjp_args, {f}));' for f, _ in cls._fields_]
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


def test_deform_input_grad_rejects_on_the_host():
    """The entry point runs the checks every field entry point runs, before any CUDA call, and names itself."""
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    lib = _lib_loaded()

    def call(p, s):
        a = ec._fill(_lib.DeformVjpArgs())
        a.loss_scale = 1024.0
        return lib.nsb_deform_input_grad(ctypes.byref(p), ctypes.byref(ec._opts()), ctypes.byref(s), ctypes.byref(a), None)

    for _, breaks, message in ec.CASES:
        p, s = ec._params(), ec._samples()
        breaks(p, s)
        assert call(p, s) != 0
        assert lib.nsb_last_error().decode() == f"nsb_deform_input_grad: {message}"
    p, s = ec._params(), ec._samples()
    p.deform_packed_tb = None
    assert call(p, s) != 0 and "missing tensors" in lib.nsb_last_error().decode()


def test_observation_normals_need_the_deformation_on_the_host():
    import test_entry_checks_cpu as ec
    from nersemble_b200 import _lib
    lib = _lib_loaded()
    a = _lib.NormalsArgs()
    a.normals, a.observation_space = ec.DUMMY, 1
    rc = lib.nsb_normals_forward(ctypes.byref(ec._params()), ctypes.byref(ec._opts()), ctypes.byref(ec._samples()), ctypes.byref(a), None)
    assert rc != 0
    assert lib.nsb_last_error().decode() == "nsb_normals_forward: observation_space needs use_deformation, offsets and vjp_scratch"


def test_space_argument_is_validated_before_any_device_call():
    from nersemble_b200 import ops
    with pytest.raises(ValueError, match="space"):
        ops.field_normals(None, positions=torch.zeros(1, 3), space="world")
    with pytest.raises(ValueError, match="normals_space"):
        ops.render_rays(None, torch.zeros(1, 3), torch.ones(1, 3), None, want_normals=True, normals_space="observed")
