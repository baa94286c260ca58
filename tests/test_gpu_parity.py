"""GPU parity: the CUDA path (through the C ABI) vs the CPU oracle and the golden fixtures."""
import numpy as np
import pytest
import torch

from conftest import load_golden, native_from_oracle, oracle_params
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
def trained():
    P = oracle_params(TRAINED)
    return P, native_from_oracle(P, DEV)


def _rays(R, seed):
    from oracle.gen_golden import ring_rays
    return ring_rays(R, seed)


def _oracle_stages(P, o, d, times, ts, te, ri, w_hash, w_deform):
    with torch.no_grad():
        return pl.render(P, o, d, times, ts, te, ri, window_hash=w_hash, window_deform=w_deform, training=False)


@pytest.fixture(scope="module")
def trained_mma(trained):
    return trained[0], native_from_oracle(trained[0], DEV, tcgen05=False)


@pytest.mark.parametrize("tensor_role", ["tcgen05", "mma.sync"])
@pytest.mark.parametrize("w_hash,w_deform", [(32.0, 7.0), (1.5, 3.3), (1, 0.0), (None, None)])
def test_field_and_composite_vs_oracle(trained, trained_mma, w_hash, w_deform, tensor_role):
    """Both inference instantiations of the deformation MLP against the oracle: the wgmma role (flag name "tcgen05", the default,
    nsb_field_tensor_role_tc.inc) and the mma.sync role (NSB_TCGEN05=0; also what the training kernels run)."""
    from nersemble_b200 import ops
    P, NP = trained if tensor_role == "tcgen05" else trained_mma
    assert (getattr(NP, "_umma_src", None) is not None) == (tensor_role == "tcgen05")
    R = 40
    o, d, times, _ = _rays(R, 3)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 50, 0.011, near=0.2)      # 2000 samples: ragged last tile
    want = _oracle_stages(P, o, d, times, ts, te, ri, w_hash, w_deform)
    info = nerfacc_cpu.pack_info(ri, R)
    got = ops.render_packed(NP, o.to(DEV), d.to(DEV), times.to(DEV), ts.to(DEV), te.to(DEV), ri.to(DEV),
                            info.to(DEV), window_hash=w_hash, window_deform=w_deform, training=False)
    got = {k: v.cpu() for k, v in got.items()}
    torch.testing.assert_close(got["offsets"], want["offsets"], rtol=2e-3, atol=3e-6)
    torch.testing.assert_close(got["density"], want["density"], rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(got["rgb_samples"], want["rgb_samples"], rtol=0, atol=2e-3)
    torch.testing.assert_close(got["weights"], want["weights"], rtol=5e-3, atol=2e-5)
    # north-star tolerance: rendered RGB within 1e-3 L2 per pixel
    assert (got["rgb"] - want["rgb"]).norm(dim=-1).max() < 1e-3
    torch.testing.assert_close(got["accumulation"], want["accumulation"], rtol=0, atol=1e-3)
    torch.testing.assert_close(got["depth"], want["depth"], rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(got["deformation"], want["deformation"], rtol=5e-3, atol=1e-5)
    assert torch.equal(got["num_samples_per_ray"], want["num_samples_per_ray"])


@pytest.mark.parametrize("name", ["fixed_trained_kernel", "fixed_trained_none", "fixed_trained_reference",
                                  "occ_eval_soft", "occ_eval_whash1", "occ_train_prepass"])
def test_render_vs_reference_goldens(name):
    """Goldens come from the REAL reference glue (oracle/gen_golden.py); all precision modes of
    the reference path must be within the 1e-3 RGB L2 tolerance of the CUDA path."""
    from nersemble_b200 import ops
    g, meta = load_golden(name)
    P = oracle_params(meta["knobs"])
    NP = native_from_oracle(P, DEV)
    R = meta["R"]
    ri = g["ray_indices"]
    info = nerfacc_cpu.pack_info(ri, R)
    got = ops.render_packed(NP, g["origins"].to(DEV), g["directions"].to(DEV), g["times"].to(DEV),
                            g["t_starts"].to(DEV), g["t_ends"].to(DEV), ri.to(DEV), info.to(DEV),
                            window_hash=meta["w_hash"], window_deform=meta["w_deform"], training=meta["training"])
    got = {k: v.cpu() for k, v in got.items()}
    l2 = (got["rgb"] - g["rgb"]).norm(dim=-1)
    assert l2.max() < 1e-3, (name, l2.max())
    torch.testing.assert_close(got["accumulation"], g["accumulation"], rtol=0, atol=2e-3)
    torch.testing.assert_close(got["depth"], g["depth"], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(got["weights"], g["weights"], rtol=2e-2, atol=1e-4)


def test_hash_blend_component(trained):
    from nersemble_b200 import ops
    P, NP = trained
    Precision.mode = "none"
    g = torch.Generator().manual_seed(5)
    n = 1000
    x = torch.rand((n, 3), generator=g) * 0.999 + 0.0005
    x[0] = 0.0; x[1] = torch.tensor([0.99999, 0.5, 0.00001])
    codes = torch.randn((n, 32), generator=g) * 0.2
    for w in (None, 12.5, 1):
        with torch.no_grad():
            want = pl.hash_ensemble(P, x, codes, w)
        got = ops.hash_blend_forward(NP, x.to(DEV), codes.to(DEV), window_hash=w, out_half=False).cpu()
        # blend weights are fp16 B-operands of the tensor-core member reduction (fp32 accumulate), like the
        # reference (hash_ensemble.py:155 casts the code to half): error budget 2^-11 per member weight
        assert ((got - want).abs().max() / want.abs().max()) < 2e-3


def test_density_fn_vs_oracle_and_golden(trained):
    from nersemble_b200 import ops
    P, NP = trained
    g, meta = load_golden("density_fn_kernel")
    got = ops.field_forward(NP, window_hash=meta["w_hash"], window_deform=meta["w_deform"],
                            positions=g["positions"].to(DEV), sample_times=g["times"].to(DEV),
                            want=("sigma",))["sigma"].cpu()
    assert (got[g["density"][:, 0] == 0] == 0).all()
    torch.testing.assert_close(got[:, None], g["density"], rtol=5e-3, atol=1e-5)


def test_march_fixed_bit_exact(trained):
    from nersemble_b200 import ops
    P, _ = trained
    o, d, _, _ = _rays(64, 9)
    d[3] = torch.tensor([0.0, 0.0, -1.0]); o[3] = torch.tensor([0.1, 0.2, 9.0])     # axis-parallel ray
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 33, 0.011, near=0.2)
    gts, gte, gri, info = ops.march_fixed(o.to(DEV), d.to(DEV), P.aabb, 33, 0.011, 0.2)
    assert torch.equal(gts.cpu(), ts) and torch.equal(gte.cpu(), te) and torch.equal(gri.cpu().long(), ri)
    assert torch.equal(info.cpu(), nerfacc_cpu.pack_info(ri, 64))


@pytest.mark.parametrize("levels", [1, 2])
def test_march_occupancy_bit_exact(trained, levels):
    from nersemble_b200 import ops
    from oracle.gen_golden import blob_grid
    P, _ = trained
    R = 96
    o, d, _, _ = _rays(R, 11)
    d[5] = torch.tensor([0.0, 0.0, -1.0]); o[5] = torch.tensor([0.1, 0.2, 9.0])
    o[6] = torch.tensor([50.0, 50.0, 50.0]); d[6] = torch.tensor([0.0, 1.0, 0.0])   # misses the box
    occ = torch.stack([blob_grid(20 + l) for l in range(levels)])
    occ[0, :, :, 64:] |= blob_grid(7)[:, :, 64:]
    aabbs = torch.stack([nerfacc_cpu._enlarge_aabb(P.aabb.reshape(-1), 2 ** l) for l in range(levels)])
    gen = torch.Generator().manual_seed(2)
    near = torch.full((R,), 0.2) + torch.rand((R,), generator=gen) * 0.011
    far = torch.full((R,), 1e3)
    ts, te, ri = nerfacc_cpu.traverse_grids(o, d, occ, aabbs, near, far, 0.011, 0.0)
    gts, gte, gri, info = ops.march_occupancy(o.to(DEV), d.to(DEV), near.to(DEV), far.to(DEV), occ.to(DEV),
                                              aabbs.to(DEV), 0.011, 0.0)
    assert gts.shape == ts.shape, (gts.shape, ts.shape)
    assert torch.equal(gri.cpu().long(), ri)
    assert torch.equal(gts.cpu(), ts) and torch.equal(gte.cpu(), te)
    assert torch.equal(info.cpu(), nerfacc_cpu.pack_info(ri, R))
    assert ts.numel() > 1000


def test_visibility_mask(trained):
    from nersemble_b200 import ops
    g = torch.Generator().manual_seed(4)
    cnt = torch.randint(0, 90, (50,), generator=g); cnt[7] = 0
    ri = torch.repeat_interleave(torch.arange(50), cnt)
    n = ri.numel()
    ts = torch.rand((n,), generator=g); te = ts + 0.011
    sig = torch.rand((n,), generator=g) * 30
    info = nerfacc_cpu.pack_info(ri, 50)
    want = nerfacc_cpu.render_visibility_from_density(ts, te, sig, packed_info=info, early_stop_eps=1e-2, alpha_thre=5e-2)
    mask, kept = ops.visibility_mask(info.to(DEV), ts.to(DEV), te.to(DEV), sig.to(DEV), 1e-2, 5e-2)
    diff = (mask.cpu() != want).sum().item()
    assert diff <= 2, diff   # thresholds can flip on 1-ulp differences of exp()
    assert abs(int(kept.sum().item()) - int(want.sum().item())) <= 2


def test_edge_cases(trained):
    from nersemble_b200 import ops
    P, NP = trained
    # empty
    e = torch.empty((0,), device=DEV)
    out = ops.field_forward(NP, window_hash=32.0, window_deform=7.0, positions=torch.empty((0, 3), device=DEV),
                            sample_times=e, want=("sigma",))
    assert out["sigma"].numel() == 0
    # a single sample, and points exactly on / outside the box faces -> selector zeroes density
    lo, hi = P.aabb[0], P.aabb[1]
    pts = torch.stack([lo, hi, (lo + hi) / 2, lo - 1.0, hi + 1.0]).to(DEV)
    sg = ops.field_forward(NP, window_hash=32.0, window_deform=None, use_deformation=False, positions=pts,
                           sample_times=torch.zeros(5, device=DEV), want=("sigma",))["sigma"].cpu()
    assert sg[0] == 0 and sg[1] == 0 and sg[3] == 0 and sg[4] == 0 and sg[2] > 0
    one = ops.field_forward(NP, window_hash=32.0, window_deform=7.0, positions=pts[2:3],
                            sample_times=torch.zeros(1, device=DEV), want=("sigma", "rgb", "offsets"))
    assert torch.isfinite(one["sigma"]).all() and one["rgb"].shape == (1, 3)
    # rays with zero samples composite to the white background
    info = torch.tensor([[0, 0], [0, 3], [3, 0]], device=DEV)
    c = ops.composite(info, torch.tensor([1., 2, 3], device=DEV), torch.tensor([2., 3, 4], device=DEV),
                      torch.tensor([0.5, 0.5, 0.5], device=DEV), torch.rand(3, 3, device=DEV))
    assert torch.equal(c["rgb"][0].cpu(), torch.ones(3)) and c["accumulation"][2].item() == 0


def test_size_independent_properties_at_full_size():
    """BASELINE config-2 sizes (2^19 tables x 32 members, 4096 rays x 256 samples): properties that
    need no oracle -- composite of a constant-density medium, linearity of the blend in the code,
    w_hash=1 equals the member-0-only table, determinism."""
    from nersemble_b200 import ops
    P = oracle_params(dict(seed=19980801, n_timesteps=4, log2_hashmap_size=19, table_scale=0.5,
                           time_std_scale=100.0, deform_last_scale=1e-3))
    NP = native_from_oracle(P, DEV)
    g = torch.Generator().manual_seed(1)
    n = 1 << 16
    x = torch.rand((n, 3), generator=g).to(DEV)
    c1 = torch.randn((n, 32), generator=g).to(DEV); c2 = torch.randn((n, 32), generator=g).to(DEV)
    f1 = ops.hash_blend_forward(NP, x, c1, out_half=False); f2 = ops.hash_blend_forward(NP, x, c2, out_half=False)
    f12 = ops.hash_blend_forward(NP, x, 2 * c1 - 3 * c2, out_half=False)
    lin = 2 * f1 - 3 * f2                                                         # linearity in the code
    assert ((f12 - lin).abs().max() / lin.abs().max()) < 3e-3                     # (fp16 blend weights)
    fa = ops.hash_blend_forward(NP, x, c1, out_half=False)
    assert torch.equal(fa, f1)                                                   # deterministic
    onehot = torch.zeros((n, 32), device=DEV); onehot[:, 0] = 1
    fw1 = ops.hash_blend_forward(NP, x, c1, window_hash=1, out_half=False)       # w==1: ones-code, window [1,0,..]
    fm0 = ops.hash_blend_forward(NP, x, onehot, out_half=False)
    torch.testing.assert_close(fw1, fm0, rtol=1e-5, atol=1e-6)
    # constant sigma: acc = 1 - exp(-sigma * len)
    R, S = 4096, 256
    ts = (torch.arange(S, device=DEV).float() * 0.011 + 5.0).repeat(R); te = ts + 0.011
    info = torch.stack([torch.arange(R, device=DEV) * S, torch.full((R,), S, device=DEV)], -1)
    c = ops.composite(info, ts, te, torch.full((R * S,), 0.7, device=DEV), torch.full((R * S, 3), 0.25, device=DEV))
    want_acc = 1 - np.exp(-0.7 * 0.011 * S)
    assert abs(c["accumulation"].mean().item() - want_acc) < 2e-4
    torch.testing.assert_close(c["rgb"], torch.full((R, 3), 0.25 * want_acc + 1 - want_acc, device=DEV), rtol=0, atol=3e-4)


@pytest.mark.parametrize("w_hash", [32.0, 1.5, None])
def test_frame_table_path_vs_oracle_and_per_sample_blend(trained, w_hash):
    """One timestep for the whole call (a camera frame): the member blend is hoisted into a per-frame table
    (nsb_blend_tables, float2 per entry) and the gather reads 8 B per corner.  Linear in the member features, so the
    result equals HashEnsemble.forward's per-sample blend (hash_ensemble.py:75-139) up to rounding: checked against the
    oracle at the tolerances of the per-sample path, and against that path itself."""
    from nersemble_b200 import ops
    P, NP = trained
    R = 40
    o, d, times, _ = _rays(R, 3)
    t0 = float(times[7])
    times = torch.full_like(times, t0)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, 50, 0.011, near=0.2)
    want = _oracle_stages(P, o, d, times, ts, te, ri, w_hash, 7.0)
    info = nerfacc_cpu.pack_info(ri, R)
    # the table itself: sum_m cw[m] * tables[e][m][:]
    ft = NP.frame_table(t0, w_hash, True, True)
    tsi = int(round(t0 * (P.time_emb.shape[0] - 1)))
    from nersemble_b200 import packing
    sc, bi = packing.blend_fold(w_hash, 32, True, True)
    cw = P.time_emb[tsi].float() * torch.tensor(sc) + torch.tensor(bi)
    ref_tab = torch.einsum("emf,m->ef", NP.tables.float().cpu(), cw)
    torch.testing.assert_close(ft.cpu(), ref_tab, rtol=1e-5, atol=1e-6)
    kw = dict(origins=o.to(DEV), directions=d.to(DEV), ray_times=times.to(DEV), t_starts=ts.to(DEV), t_ends=te.to(DEV),
              ray_indices=ri.to(DEV), window_hash=w_hash, window_deform=7.0)
    per_sample = ops.field_forward(NP, **kw)
    frame = ops.field_forward(NP, uniform_time=t0, **kw)
    assert torch.equal(frame["offsets"], per_sample["offsets"])                       # the deformation does not change
    torch.testing.assert_close(frame["sigma"], per_sample["sigma"], rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(frame["rgb"], per_sample["rgb"], rtol=0, atol=2e-3)
    torch.testing.assert_close(frame["sigma"].cpu(), want["density"][:, 0], rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(frame["rgb"].cpu(), want["rgb_samples"], rtol=0, atol=2e-3)
    # fused render, fixed march: per-ray outputs against the oracle (north-star tolerance 1e-3 L2 per pixel)
    got = ops.render_rays(NP, o.to(DEV), d.to(DEV), times.to(DEV), window_hash=w_hash, window_deform=7.0, sampler="fixed",
                          n_per_ray=50, near_plane=0.2, step=0.011, uniform_time=t0)
    assert (got["rgb"].cpu() - want["rgb"]).norm(dim=-1).max() < 1e-3
    torch.testing.assert_close(got["accumulation"].cpu(), want["accumulation"], rtol=0, atol=1e-3)
    torch.testing.assert_close(got["depth"].cpu(), want["depth"], rtol=1e-3, atol=1e-3)
