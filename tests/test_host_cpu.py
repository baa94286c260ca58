"""CPU tests of the host logic: packing layouts, level table, window folding, C-ABI exports."""
import ctypes
import sys
import os
import re

import numpy as np
import pytest
import torch

from nersemble_b200 import _lib, packing
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import hashgrid_levels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_level_table_matches_oracle_and_survey():
    lv = packing.level_table()
    o = hashgrid_levels()
    assert lv["res"] == [16, 24, 34, 49, 71, 102, 148, 213, 308, 446, 646, 934, 1352, 1956, 2831, 4096]
    assert lv["total_entries"] == 6299960 == o.total_entries
    assert lv["offset"][:6] == [0, 4096, 17920, 57224, 174880, 532792]
    assert lv["hashed"] == [0] * 5 + [1] * 11 == [int(h) for h in o.hashed]
    np.testing.assert_array_equal(np.array(lv["scale"], np.float32), o.scale)


def test_tables_roundtrip_and_rearrange():
    g = torch.Generator().manual_seed(0)
    grids = [torch.rand(40 * 8, generator=g) for _ in range(8)]
    t = packing.tables_from_tcnn(grids)
    assert t.shape == (40, 32, 2)
    # reference mapping (hash_ensemble.py:112): column l*8 + p*2 + f of grid c -> member c*4+p, feature f
    assert t[7, 2 * 4 + 3, 1] == grids[2][7 * 8 + 3 * 2 + 1]
    back = packing.tables_to_tcnn(t)
    for a, b in zip(grids, back):
        assert torch.equal(a, b)
    assert torch.equal(pl.tables_from_tcnn(grids), t)


def _brute_pack(W, colmap, group_cols):
    N, _ = W.shape
    Kp = len(colmap); Np = ((N + group_cols - 1) // group_cols) * group_cols
    out = []
    for grp in range(Np // group_cols):
        for kt in range(Kp // 16):
            for pair in range(group_cols // 16):
                for lane in range(32):
                    g, q = lane >> 2, lane & 3
                    for ntsel in range(2):
                        n = grp * group_cols + pair * 16 + ntsel * 8 + g
                        for hi in range(2):
                            for e in range(2):
                                k = kt * 16 + hi * 8 + 2 * q + e
                                c = colmap[k]
                                out.append(float(W[n, c]) if (c >= 0 and n < N) else 0.0)
    return torch.tensor(out).half()


def test_pack_mma_b_matches_fragment_definition():
    g = torch.Generator().manual_seed(1)
    W = torch.randn((6, 32), generator=g)
    cm = list(range(31, -1, -1)); cm[5] = -1
    assert torch.equal(packing.pack_mma_b(W, cm, 16), _brute_pack(W, cm, 16))
    W = torch.randn((128, 40), generator=g)
    cm = [(-1 if k % 7 == 0 else k % 40) for k in range(48)]
    assert torch.equal(packing.pack_mma_b(W, cm, 64), _brute_pack(W, cm, 64))


def test_colmaps_are_consistent_with_reference_orders():
    cm = packing.deform_input_colmap()
    assert len(cm) == 176 and sorted(c for c in cm if c >= 0) == list(range(173))
    assert cm[0] == 0 and cm[1] == 21            # (sin, cos) of x*f0
    assert cm[2 * 7] == 7 and cm[2 * 7 + 1] == 28  # y*f0
    assert cm[42:46] == [42, 43, 44, -1]
    hm = packing.head_input_colmap()
    assert sorted(hm) == list(range(32)) and hm[16:19] == [0, 1, 2] and hm[1] == 3


def test_pack_sizes():
    P = pl.random_params(n_timesteps=2, log2_hashmap_size=4)
    dp, db = packing.pack_deform(P.deform_w, P.deform_b, P.r_w, P.r_b, P.v_w, P.v_b)
    assert dp.numel() * 2 == 258048 and db.numel() == 776
    assert packing.pack_field(P.base_w, P.head_w).numel() * 2 == 20480


def test_blend_fold_matches_reference_semantics():
    code = torch.randn(5, 32)
    for w in (None, 1, 1.25, 1.999, 2.0, 7.3, 32.0):
        sc, bi = packing.blend_fold(w)
        cw = code * torch.tensor(sc) + torch.tensor(bi)
        P = pl.random_params(n_timesteps=2, log2_hashmap_size=4)
        c2, win = pl.blend_code(P, code, w)
        want = c2 if win is None else c2 * win[None]
        torch.testing.assert_close(cw, want, rtol=1e-6, atol=1e-7)


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "nsb.h")).read()
    declared = set(re.findall(r"\b(nsb_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.nsb_version() == 200
    lib.nsb_deform_packed_bytes.restype = ctypes.c_size_t
    lib.nsb_field_packed_bytes.restype = ctypes.c_size_t
    assert lib.nsb_deform_packed_bytes() == 94 * 2048 and lib.nsb_field_packed_bytes() == 20480


def test_ops_refuse_cpu_tensors():
    from nersemble_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.march_fixed(torch.zeros(2, 3), torch.ones(2, 3), torch.tensor([[0., 0, 0], [1, 1, 1]]), 4, 0.1)


def test_time_bias_packing_is_the_same_linear_map():
    """pack_deform_tb: W_code . code[t] + b moved into a per-timestep bias; layer-0 pre-activation unchanged."""
    P = pl.random_params(n_timesteps=5, log2_hashmap_size=4)
    packed, cb = packing.pack_deform_tb(P.deform_w, P.deform_b, P.r_w, P.r_b, P.v_w, P.v_b, P.time_emb_deform)
    assert packed.numel() * 2 == 94 * 2048 and cb.shape == (5, 2, 128)
    h = lambda t: t.half().float()
    enc = torch.randn(7, 45)
    for l in (0, 4):
        W, b = P.deform_w[l], P.deform_b[l]
        for t in range(5):
            x = torch.cat([enc, P.time_emb_deform[t][None].expand(7, -1)], -1)
            full = h(x) @ h(W[:, :173]).t() + b
            split = h(enc) @ h(W[:, :45]).t() + cb[t, 0 if l == 0 else 1]
            torch.testing.assert_close(split, full, rtol=1e-5, atol=1e-6)


def test_gather_plans_reproduce_the_packers():
    """Training re-packs the MLP weights every step through cached gather plans (packing.gather_plan); they must give
    exactly what the defining packers give."""
    from nersemble_b200 import packing as pk
    g = torch.Generator().manual_seed(0)
    stem = [torch.randn(s, generator=g) for s in pk._STEM_SHAPES]
    sb = [torch.randn(128, generator=g) for _ in range(6)]
    r_w, v_w, r_b, v_b = torch.randn(3, 128, generator=g), torch.randn(3, 128, generator=g), torch.randn(3, generator=g), torch.randn(3, generator=g)
    codes = torch.randn(4, 128, generator=g)
    for _ in range(2):      # second pass uses the cached plans
        b, c = pk.pack_deform_weights_fast(stem, r_w, v_w)
        assert torch.equal(b, pk.pack_deform_tb(stem, sb, r_w, r_b, v_w, v_b, codes)[0])
        assert torch.equal(c, pk.pack_deform_bwd(stem, r_w, v_w))
        bw = [torch.randn(64, 32, generator=g), torch.randn(16, 64, generator=g)]
        hw = [torch.randn(64, 32, generator=g), torch.randn(64, 64, generator=g), torch.randn(16, 64, generator=g)]
        f, fb = pk.pack_field_fast(bw, hw)
        assert torch.equal(f, pk.pack_field(bw, hw)) and torch.equal(fb, pk.pack_field_bwd(bw, hw))
        al = pk.pack_all_fast(stem, r_w, v_w, bw, hw)      # one gather for all four
        assert len(al) == 4
        for got, want in zip(al, (b, c, f, fb)):
            assert torch.equal(got, want)
    assert torch.equal(pk.deform_bias_vector(sb, r_b, v_b), pk.pack_deform(stem, sb, r_w, r_b, v_w, v_b)[1])


def test_pack_deform_umma_layout():
    """wgmma B operands (packing.pack_deform_umma): 14 blocks per tile in order of use, [n x 64 k] in K-major
    no-swizzle core-matrix order -- byte offset (n/8)*1024 + (k/8)*128 + (n%8)*16 + (k%8)*2 (descriptor LBO 128, SBO 1024);
    K = the reference's encoding column order, zero padded; the gather-plan version is identical."""
    from nersemble_b200 import packing as pk
    g = torch.Generator().manual_seed(1)
    stem = [torch.randn(s, generator=g) for s in pk._STEM_SHAPES]
    r_w, v_w = torch.randn(3, 128, generator=g), torch.randn(3, 128, generator=g)
    a = pk.pack_deform_umma(stem, r_w, v_w)
    assert a.dtype == torch.float16 and a.numel() * 2 == 12 * 16384 + 2 * 2048
    assert torch.equal(a, pk.pack_deform_umma_fast(stem, r_w, v_w))
    el = lambda blk, n, k: float(a[blk * 8192 + (n // 8) * 512 + (k // 8) * 64 + (n % 8) * 8 + (k % 8)])
    h = lambda x: float(x.half())
    assert el(0, 37, 21) == h(stem[0][37, 21]) and el(0, 37, 45) == 0.0 and el(0, 127, 44) == h(stem[0][127, 44])
    assert el(1, 5, 63) == h(stem[1][5, 63]) and el(2, 5, 0) == h(stem[1][5, 64])            # layer 1: two 64-wide K blocks
    assert el(7, 9, 3) == h(stem[4][9, 173 + 3]) and el(8, 9, 3) == h(stem[4][9, 173 + 67])    # layer 4: hidden columns first
    assert el(9, 9, 44) == h(stem[4][9, 44]) and el(9, 9, 47) == 0.0                         # ... then the posenc columns
    assert el(10, 100, 7) == h(stem[5][100, 7])
    heads = lambda half, n, k: float(a[12 * 8192 + half * 1024 + (n // 8) * 512 + (k // 8) * 64 + (n % 8) * 8 + (k % 8)])
    assert heads(0, 1, 5) == h(v_w[1, 5]) and heads(0, 4, 5) == h(r_w[1, 5]) and heads(1, 4, 5) == h(r_w[1, 69])
    assert heads(0, 6, 0) == 0.0 and heads(1, 15, 63) == 0.0


def test_forward_kernel_gather_role_has_no_spill_storm():
    """Regression guard for a performance cliff, not for correctness: local-memory traffic inside the gather
    role of field_kernel_ws is catastrophic (a spill inside the sample loop costs more than the loop's own work)
    and ptxas allocates that role erratically.  The committed source builds with <= 9 STL/LDL there; fail loudly when a
    change (or a different toolkit) pushes a variant over 16."""
    import shutil, subprocess
    obj = os.path.join(ROOT, "nersemble_b200", "csrc", "nsb_field.o")
    if not os.path.exists(obj) or shutil.which("cuobjdump") is None:
        pytest.skip("needs the in-tree object file and cuobjdump")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "spill_report.py"), obj], capture_output=True, text=True).stdout
    rows = [l.split() for l in out.splitlines() if "gather" in l]
    assert len(rows) >= 12
    for r in rows:
        assert int(r[r.index("gather") + 1]) <= 16, out
    # the wgmma instantiations (the default for inference): the committed source builds with at most 2 spill instructions
    # in the gather role
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "spill_report.py"), obj, "kernel_tc"], capture_output=True, text=True).stdout
    rows = [l.split() for l in out.splitlines() if "gather" in l]
    assert len(rows) >= 8
    for r in rows:
        assert int(r[r.index("gather") + 1]) <= 12, out


def test_ctypes_structs_match_the_c_header_layout(tmp_path):
    """ABI drift guard: size and every field offset of the ctypes mirrors in _lib.py against what a C compiler makes of
    include/nsb.h (the header is plain C; gcc is in the image)."""
    import shutil, subprocess
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc")
    pairs = {"nsb_levels": _lib.Levels, "nsb_field_params": _lib.FieldParams, "nsb_field_opts": _lib.FieldOpts,
             "nsb_samples": _lib.Samples, "nsb_field_out": _lib.FieldOut, "nsb_field_bwd_args": _lib.FieldBwdArgs,
             "nsb_table_adam_args": _lib.TableAdamArgs, "nsb_loss_args": _lib.LossArgs,
             "nsb_composite_args": _lib.CompositeArgs, "nsb_deform_bwd_args": _lib.DeformBwdArgs,
             "nsb_render_args": _lib.RenderArgs, "nsb_render_ws_header": _lib.RenderWsHeader,
             "nsb_vis_compact_args": _lib.VisCompactArgs, "nsb_ray_batch_args": _lib.RayBatchArgs,
             "nsb_composite_bwd_args": _lib.CompositeBwdArgs, "nsb_march_args": _lib.MarchArgs}
    header = open(os.path.join(ROOT, "include", "nsb.h")).read()
    assert set(re.findall(r"^typedef struct (nsb_\w+)", header, flags=re.M)) == set(pairs)     # every struct is mirrored
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nsb.h"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    want = {}
    for cname, cls in pairs.items():
        want[(cname, "size")] = ctypes.sizeof(cls)
        for fname, _ in cls._fields_:
            want[(cname, fname)] = getattr(cls, fname).offset
    got = {(a, b): int(c) for a, b, c in (l.split() for l in out.splitlines())}
    assert got == want, {k: (got.get(k), want.get(k)) for k in set(got) | set(want) if got.get(k) != want.get(k)}


def test_rank1_slot_map_for_many_timesteps():
    """The rank-1 table-gradient scatter keys its workspace by timestep SLOT: identity for <= 32 timesteps, the batch's
    distinct timesteps (same rounding as the kernels: round(t * (T - 1))) for longer sequences, and no rank-1 path when a
    batch holds more than 32 distinct timesteps or per-sample blend codes are given."""
    from types import SimpleNamespace
    from nersemble_b200 import ops
    dev = torch.device("cpu")
    slot, n = ops._rank1_slots(SimpleNamespace(n_timesteps=24), dev, {})
    assert n == 24 and torch.equal(slot, torch.arange(24, dtype=torch.int32))
    T = 200
    steps = torch.tensor([3, 3, 77, 199, 0, 77])
    times = steps.float() / (T - 1)
    slot, n = ops._rank1_slots(SimpleNamespace(n_timesteps=T), dev, {"origins": torch.zeros(6, 3), "ray_times": times})
    assert n == 4 and slot.shape == (T,)
    assert sorted(slot[[0, 3, 77, 199]].tolist()) == [0, 1, 2, 3] and int((slot >= 0).sum()) == 4
    many = torch.arange(40).float() / (T - 1)
    assert ops._rank1_slots(SimpleNamespace(n_timesteps=T), dev, {"origins": torch.zeros(40, 3), "ray_times": many}) == (None, 0)
    assert ops._rank1_slots(SimpleNamespace(n_timesteps=24), dev, {"sample_blend_codes": torch.zeros(5, 32)}) == (None, 0)
    # explicit positions use per-sample times
    slot, n = ops._rank1_slots(SimpleNamespace(n_timesteps=T), dev, {"positions": torch.zeros(3, 3), "sample_times": times[:3]})
    assert n == 2


def test_posenc_sine_reduction_constants():
    """tc::sin_reduced (nsb_tc.cuh) = two-constant Cody-Waite reduction to [-pi, pi] + MUFU.SIN, the posenc of the wgmma
    deformation role.  Emulated in numpy (fp32 operands, the FMA's exact product in float64): over the argument range of
    the encoding -- fl(2 pi p) * 2^j for j < 7 and positions up to 4 box widths outside the box -- the REDUCTION moves the
    sine by < 2e-7 (MUFU.SIN adds < 4e-7 on the reduced range); the value then becomes an fp16 MMA operand
    (spacing 4.9e-4 near 1), as in the oracle's kernel mode."""
    import numpy as np
    rng = np.random.default_rng(0)
    p = rng.uniform(-4.0, 5.0, size=200000).astype(np.float32)
    a = (np.float32(6.283185307179586) * p).astype(np.float32)
    worst = 0.0
    for j in range(7):
        for shift in (np.float32(0.0), np.float32(1.5707963267948966)):
            x = (a * np.float32(1 << j) + shift).astype(np.float32)
            k = np.rint((x * np.float32(0.15915494309189535)).astype(np.float32)).astype(np.float32)
            r = (x.astype(np.float64) - k.astype(np.float64) * np.float64(np.float32(6.2831854820251465))).astype(np.float32)
            r = (r.astype(np.float64) - k.astype(np.float64) * np.float64(np.float32(-1.7484555314695172e-07))).astype(np.float32)
            assert np.abs(r).max() < 3.1416 + 1e-3
            worst = max(worst, float(np.abs(np.sin(r.astype(np.float64)) - np.sin(x.astype(np.float64))).max()))
    assert worst < 2e-7, worst
