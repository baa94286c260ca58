"""The inference render kernels in their steady state: the benchmark's batch (4096 rays x 256 samples = 2^20 samples,
8192 tiles, ~62 tiles per CTA on 132 SMs), two ragged fixed-stride batches and an occupancy-grid batch, so that every
CTA of the persistent kernels runs at least 8 tiles.  From a CTA's third tile on, the wgmma pipeline reuses the shared
buffers of tile i - 2 without a barrier of its own (nsb_field_tensor_role_tc.inc), its feat_full parity flips back,
the prefetch runs two tiles ahead and the weight ring runs through my_tiles * kTcBlocksPerTile blocks; the other render
tests give each CTA at most two tiles.  Checked here, on every kernel render_rays reaches:

  1. per-sample and per-ray outputs of one launch are bit-identical to launches on consecutive ray chunks of at most
     min(64, SMS / 2) tiles (one tile per CTA: the regime the small tests pin to the oracle);
  2. the samples of the tiles the small tests never reach (iterations 2 and 3 of a CTA, its last two iterations, the
     ragged last tile) against the CPU oracle on the kernel's own packed samples;
  3. every ray of the full launch against the float64 composite of the launch's own per-sample values, within the
     float32 rounding bound of scan_oracle, and the depth clip range exactly;
  4. the timestep-stack, line-gather and mma.sync kernels against each other at full scale;
  5. two launches of the benchmark path are bit-identical.

Each bounded check (2, 3) is shown on the reference side to reject a stale tile buffer and rows shifted by one by at
least 10x.  The tile -> (CTA, iteration) map is render_scale_oracle's: tile k runs on CTA k % SMS as its iteration
k // SMS."""
import pytest
import torch

import render_scale_oracle as rso
import scan_oracle as so
from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FULL = dict(seed=19980801, n_timesteps=24, log2_hashmap_size=19, table_scale=0.5, time_std_scale=100.0,
            deform_last_scale=1e-3)
W_DEFORM, STEP, NEAR = 7.0, 0.011, 0.2
T_UNIFORM = 13 / 23                    # the frame kernels: one captured timestep for every ray
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 0
CHUNK_SAMPLES = min(64, SMS // 2) * 128 if SMS else 64 * 128
MAX_PROBE_RAYS = 96
R_OCC = 16384                          # the plugin's frame path renders >= 16 384 rays with one uniform time
# the config-2 tolerances of test_gpu_fullsize.test_full_size_oracle_parity_config2_shape: (rtol, atol)
TOL = dict(offsets=(4e-3, 3e-6), density=(5e-3, 1e-5), rgb_samples=(0.0, 2e-3), weights=(5e-3, 2e-5),
           accumulation=(0.0, 1e-3), depth=(1e-3, 1e-3), deformation=(5e-3, 1e-5))
RGB_L2 = 1e-3

# fixed-stride batches: the benchmark's, and two ragged ones found from the SM count (n_per_ray odd, so rays start
# mid-tile): the last tile 1 row with n_tiles = 1 mod SMS (one CTA runs one tile more than the others), and the last
# tile 65 rows with n_tiles = -1 mod SMS (all CTAs but one run the extra tile)
SHAPES = {"A": (4096, 256)}
if SMS:
    SHAPES["B1"] = rso.ragged_batch(SMS, 1, 1, range(129, 256, 2))
    SHAPES["B65"] = rso.ragged_batch(SMS, 65, SMS - 1, range(129, 256, 2))
    # what the batches have to reach on this device, or the paths this file exists for are not covered
    for _name, (_R, _S) in SHAPES.items():
        assert min(rso.tiles_per_cta(_R * _S, SMS)) >= 8, f"shape {_name}: fewer than 8 tiles per CTA"
    assert rso.n_tiles(CHUNK_SAMPLES) <= SMS, "a chunk must give every CTA at most one tile"

# kernel -> (render_rays keywords, time mode, NativeParams flavour).  The template each one reaches (nsb_field.cu):
KERNELS = {
    "stack": (dict(), "mixed", "tc"),                                              # render_kernel_tc<4, true, true>
    "line": (dict(line_gather=True), "mixed", "tc"),                               # render_kernel_tc<4, false, false>
    "frame": (dict(uniform_time=T_UNIFORM), "uniform", "tc"),                      # render_kernel_tc<4, true, false>
    "lerp_stack": (dict(time_interpolation="linear"), "lerp", "tc"),               # render_kernel_tc_lerp<4, true, true>
    "lerp_line": (dict(time_interpolation="linear", line_gather=True), "lerp", "tc"),   # render_kernel_tc_lerp<4, false, false>
    "mma_sync": (dict(), "mixed", "ws"),                                           # render_kernel_ws<true, 0>
    "no_deform": (dict(use_deformation=False), "none", "tc"),                      # render_kernel_ws<false, 0>
    "occ_stack": (dict(), "mixed", "tc"),                                          # render_kernel_tc<2, true, true>
    "occ_frame": (dict(uniform_time=T_UNIFORM), "uniform", "tc"),                  # render_kernel_tc<2, true, false>
}
# (kernel, shape, w_hash): every fixed-stride kernel on every fixed shape at w_hash = 32 (one-hot blend), the
# benchmark path also at w_hash = 1.5 (a blend of two members), the occupancy kernels on their own batch
CASES = ([(k, s, 32.0) for s in ("A", "B1", "B65") for k in KERNELS if not k.startswith("occ")] + [("stack", "A", 1.5)] +
         [("occ_stack", "OCC", 32.0), ("occ_frame", "OCC", 32.0)])
CASE_IDS = [f"{k}-{s}-w{w:g}" for k, s, w in CASES]
ORACLE_CASES = [c for c in CASES if KERNELS[c[0]][1] != "none"]


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


@pytest.fixture(autouse=True, scope="module")
def _free_module_caches():
    yield
    for c in (_NP, _RAYS, _FULL, _CHUNKED, _ORACLE):
        c.clear()
    torch.cuda.empty_cache()


_NP, _RAYS, _FULL, _CHUNKED, _ORACLE = {}, {}, {}, {}, {}


def _params(flavour="tc"):
    if flavour not in _NP:
        P = oracle_params(FULL)
        _NP[flavour] = (P, native_from_oracle(P, DEV, tcgen05=False if flavour == "ws" else None))
    return _NP[flavour]


def _edge_rays(o, d, spots, aabb):
    """test_full_size_oracle_parity_config2_shape's rays at the given (late) ray indices: one grazing the x = max face,
    one running along an edge, one missing the box."""
    lo, hi = aabb[0], aabb[1]
    o[spots[0]] = torch.tensor([float(hi[0]) - 1e-4, 0.2, 9.0]); d[spots[0]] = torch.tensor([0.0, 0.0, -1.0])
    o[spots[1]] = torch.tensor([float(lo[0]), float(lo[1]), 9.0]); d[spots[1]] = torch.tensor([0.0, 0.0, -1.0])
    o[spots[2]] = torch.tensor([50.0, 50.0, 50.0]); d[spots[2]] = torch.tensor([0.0, 1.0, 0.0])


def _rays(shape):
    """ring_rays with every timestep present (rays 0..23 at k / 23, the rest unsorted, fractional) and the edge rays in
    late tiles: the rays under the first row of the last tile of CTA 0, of a middle CTA and of the last CTA (fixed stride), or
    near the end of the batch (occupancy).  Returns (o, d, times, edge ray ids) on the device."""
    if shape not in _RAYS:
        from oracle.gen_golden import ring_rays
        P, _ = _params()
        R = R_OCC if shape == "OCC" else SHAPES[shape][0]
        o, d, times, _ = ring_rays(R, 17)
        times[:24, 0] = torch.arange(24) / 23.0
        if shape == "OCC":
            spots = [R - 1500, R - 700, R - 1]
        else:
            S = SHAPES[shape][1]
            mt = rso.tiles_per_cta(R * S, SMS)
            last = max(c for c in range(SMS) if mt[c] > 0)
            spots = []
            for c in (0, last // 2, last):
                r = rso.tile_of(c, mt[c] - 1, SMS) * rso.TILE // S
                while r in spots:          # two of the tiles lie on one ray: the ray before it
                    r -= 1
                spots.append(r)
        assert len(set(spots)) == 3 and min(spots) >= 24
        _edge_rays(o, d, spots, P.aabb)
        _RAYS[shape] = (o.to(DEV), d.to(DEV), times.to(DEV), spots)
    return _RAYS[shape]


def _occ_grid(NP):
    from oracle.gen_golden import blob_grid
    return blob_grid(5)[None].to(DEV), torch.tensor(NP.aabb_list, device=DEV).reshape(1, 6)


def _render(kernel, shape, wh, o, d, t):
    from nersemble_b200 import ops
    kw, mode, flavour = KERNELS[kernel]
    _, NP = _params(flavour)
    if mode == "uniform":
        t = torch.full_like(t, T_UNIFORM)
    if shape == "OCC":
        b, ab = _occ_grid(NP)
        R = o.shape[0]
        return ops.render_rays(NP, o, d, t, window_hash=wh, window_deform=W_DEFORM, sampler="occupancy",
                               near_planes=torch.full((R,), NEAR, device=DEV), far_planes=torch.full((R,), 1e3, device=DEV),
                               binaries=b, aabbs=ab, step=STEP, **kw)
    return ops.render_rays(NP, o, d, t, window_hash=wh, window_deform=W_DEFORM, sampler="fixed",
                           n_per_ray=SHAPES[shape][1], near_plane=NEAR, step=STEP, **kw)


def _clip_range(res):
    """The launch's depth clip range from its workspace header (depth_range[2], ordered uint32) as floats; (1, 1)
    when the launch had no sample, as render_composite_phase does."""
    h = res["_buffers"]["header"][:2].view(torch.int32).tolist()          # barrier, depth_range[0..1], status
    lo_u, hi_u = h[1] & 0xffffffff, h[2] & 0xffffffff
    if lo_u == 0xffffffff:
        return 1.0, 1.0
    return rso.ordered_to_float(lo_u), rso.ordered_to_float(hi_u)


PER_RAY = ("rgb", "accumulation", "depth", "deformation", "num_samples_per_ray", "packed_info")
PACKED = ("t_starts", "t_ends", "ray_indices", "sigma", "rgb", "offsets", "weights")


def _outputs(res):
    out = {k: res[k] for k in PER_RAY if k in res}
    out["packed"] = res.packed()
    out["clip"] = _clip_range(res)
    return out


def _full(case):
    if case not in _FULL:
        kernel, shape, wh = case
        o, d, t, _ = _rays(shape)
        _FULL[case] = _outputs(_render(kernel, shape, wh, o, d, t))
    return _FULL[case]


def _counts(shape):
    """Samples per ray of the batch, for the chunker: the fixed stride, or march_occupancy's counts (the two-pass
    marcher is bit-identical to the fused march, test_gpu_render.py)."""
    o, d, t, _ = _rays(shape)
    if shape != "OCC":
        return torch.full((o.shape[0],), SHAPES[shape][1], dtype=torch.long)
    from nersemble_b200 import ops
    b, ab = _occ_grid(_params()[1])
    R = o.shape[0]
    _, _, _, info = ops.march_occupancy(o, d, torch.full((R,), NEAR, device=DEV), torch.full((R,), 1e3, device=DEV),
                                        b, ab, STEP, 0.0)
    return info[:, 1].cpu()


def _chunked(case):
    """The same rays in consecutive chunks of at most CHUNK_SAMPLES samples, outputs concatenated (packed ray indices
    and packed_info offsets shifted to the whole batch), plus each ray's chunk clip range."""
    if case not in _CHUNKED:
        kernel, shape, wh = case
        o, d, t, _ = _rays(shape)
        counts = _counts(shape)
        parts, lo, hi = [], [], []
        base = 0
        for a, b in rso.chunk_rays(counts, CHUNK_SAMPLES):
            r = _outputs(_render(kernel, shape, wh, o[a:b], d[a:b], t[a:b]))
            r["packed"]["ray_indices"] = r["packed"]["ray_indices"] + a
            r["packed_info"] = r["packed_info"] + torch.tensor([base, 0], device=DEV)
            base += int(counts[a:b].sum())
            parts.append(r)
            lo.append(torch.full((b - a,), r["clip"][0])); hi.append(torch.full((b - a,), r["clip"][1]))
        out = {k: torch.cat([p[k] for p in parts]) for k in PER_RAY if k in parts[0]}
        out["packed"] = {k: torch.cat([p["packed"][k] for p in parts]) for k in parts[0]["packed"]}
        out["clip_lo"], out["clip_hi"] = torch.cat(lo).to(DEV), torch.cat(hi).to(DEV)
        out["n_chunks"] = len(parts)
        _CHUNKED[case] = out
    return _CHUNKED[case]


def _where(bad: torch.Tensor) -> str:
    """Where the flagged samples ran: (tile, CTA, iteration) of the first few and the iterations they fall in."""
    s = torch.nonzero(bad.reshape(bad.shape[0], -1).any(1)).flatten().cpu()
    tiles = torch.unique(s // rso.TILE).tolist()
    places = [(t,) + rso.tile_place(t, SMS) for t in tiles[:8]]
    its = sorted(set(rso.tile_place(t, SMS)[1] for t in tiles))
    return f"{s.numel()} samples in {len(tiles)} tiles; first (tile, CTA, it): {places}; iterations {its[:20]}"


def _report(what, value, bound=None):
    print(f"  {what}: {value:.3e}" + ("" if bound is None else f"  (bound {bound:.3e})"), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# 1. one launch == chunked launches, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_full_launch_equals_one_tile_per_cta_chunks(case):
    """Every per-sample and per-ray output of the full launch equals the chunked launches bit for bit.  A sample's
    result depends only on its own inputs (the field phase computes every row on its own, and the composite of a ray
    runs lane-strided over that ray's samples in one warp), so neither its tile, its row nor its CTA may change a bit.
    Depth is clipped to each launch's own midpoint range, so it is compared on the rays inside both ranges; the clip
    itself is checked in test_every_ray_against_the_float64_composite."""
    full, ch = _full(case), _chunked(case)
    kernel, shape, _ = case
    n = full["packed"]["t_starts"].shape[0]
    print(f"\n{case}: {n} samples, {rso.n_tiles(n)} tiles, min tiles per CTA {min(rso.tiles_per_cta(n, SMS))}; "
          f"{ch['n_chunks']} chunks of <= {rso.n_tiles(CHUNK_SAMPLES)} tiles")
    if shape == "OCC":
        assert min(rso.tiles_per_cta(n, SMS)) >= 8, "the occupancy batch gives some CTA fewer than 8 tiles"
        assert torch.equal(full["num_samples_per_ray"].cpu(), _counts(shape))
    for k in PACKED:
        if k in full["packed"]:
            a, b = full["packed"][k], ch["packed"][k]
            assert a.shape == b.shape, (k, a.shape, b.shape)
            bad = (a != b) & ~(torch.isnan(a) & torch.isnan(b)) if a.is_floating_point() else a != b
            assert not bad.any(), f"{case} packed {k}: {_where(bad)}"
    for k in ("rgb", "accumulation", "deformation", "num_samples_per_ray", "packed_info"):
        if k in full:
            bad = (full[k] != ch[k]).reshape(full[k].shape[0], -1).any(1)
            assert not bad.any(), f"{case} {k}: rays {torch.nonzero(bad).flatten()[:8].tolist()} differ"
    lo, hi = full["clip"]
    dep_f, dep_c = full["depth"][:, 0], ch["depth"][:, 0]
    inside = (dep_f > lo) & (dep_f < hi) & (dep_c > ch["clip_lo"]) & (dep_c < ch["clip_hi"])
    bad = inside & (dep_f != dep_c)
    assert not bad.any(), f"{case} depth: rays {torch.nonzero(bad).flatten()[:8].tolist()} differ"
    print(f"  bit-identical; depth compared on {int(inside.sum())} of {inside.numel()} rays (the rest clipped)")
    assert int(inside.sum()) > 0.5 * inside.numel()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the oracle on the tiles the small tests never reach
# ---------------------------------------------------------------------------------------------------------------------
def _probe(case):
    """The probe rays of a launch (render_scale_oracle.probe_tiles / select_rays, plus the edge rays and the rays of
    tile 0, the source of the stale-buffer control) and their samples."""
    full = _full(case)
    pk = full["packed"]
    n = pk["t_starts"].shape[0]
    _, _, _, spots = _rays(case[1])
    ri = pk["ray_indices"].cpu()
    tile0 = torch.unique(ri[:rso.TILE]).tolist()
    rays, taken = rso.select_rays(ri, rso.probe_tiles(n, SMS), MAX_PROBE_RAYS, extra=list(spots) + tile0)
    idx, sub_info, local = rso.subset_samples(full["packed_info"], rays)
    return rays, taken, idx, sub_info, local


def _oracle(case, rays, idx, local):
    """pl.render on the probe rays' packed samples, once per (shape, w_hash, time mode): the kernels that render the
    same thing share it."""
    kernel, shape, wh = case
    mode = KERNELS[kernel][1]
    key = (shape, wh, mode)
    full = _full(case)
    if key not in _ORACLE:
        P, _ = _params()
        o, d, t, _ = _rays(shape)
        if mode == "uniform":
            t = torch.full_like(t, T_UNIFORM)
        ts, te = full["packed"]["t_starts"].cpu()[idx], full["packed"]["t_ends"].cpu()[idx]
        with torch.no_grad():
            want = pl.render(P, o.cpu()[rays], d.cpu()[rays], t.cpu()[rays], ts, te, local, window_hash=wh,
                             window_deform=W_DEFORM, training=False)
        _ORACLE[key] = (rays, idx, want)
    r0, i0, want = _ORACLE[key]
    assert torch.equal(r0, rays) and torch.equal(i0, idx), "kernels that share an oracle must pack the same samples"
    return want


def _lerp_reference(case, rays, idx, sub_info):
    """The per-sample-code path (test_gpu_time_interp.test_mixed_fractional_times): field_forward with each sample's
    interpolated blend and warp codes (ops.time_codes) on the probe rays' packed samples, then composite."""
    from nersemble_b200 import ops
    _, NP = _params()
    o, d, t, _ = _rays(case[1])
    pk = _full(case)["packed"]
    i = idx.to(DEV)
    ri = pk["ray_indices"][i]
    codes = ops.time_codes(NP, t)
    f = ops.field_forward(NP, origins=o, directions=d, ray_times=t.reshape(-1), t_starts=pk["t_starts"][i],
                          t_ends=pk["t_ends"][i], ray_indices=ri, window_hash=case[2], window_deform=W_DEFORM,
                          sample_blend_codes=codes["blend_codes"][ri.long()].contiguous(),
                          sample_warp_codes=codes["warp_codes"][ri.long()].contiguous())
    c = ops.composite(sub_info.to(DEV), pk["t_starts"][i], pk["t_ends"][i], f["sigma"], f["rgb"], f["offsets"])
    return {"offsets": f["offsets"].cpu(), "density": f["sigma"][:, None].cpu(), "rgb_samples": f["rgb"].cpu(),
            "weights": c["weights"].cpu(), "rgb": c["rgb"].cpu(), "accumulation": c["accumulation"].cpu(),
            "deformation": c["deformation"].cpu()}


@pytest.mark.parametrize("case", ORACLE_CASES, ids=[f"{k}-{s}-w{w:g}" for k, s, w in ORACLE_CASES])
def test_late_tiles_against_the_oracle(case):
    """The probe tiles (iterations 2 and 3, the last two iterations of CTA 0, a middle CTA and the last CTA, the ragged
    last tile, the edge rays) against pl.render on the kernel's own packed samples, at the config-2 tolerances of
    test_gpu_fullsize; the oracle's depth is the expected depth clipped to the full launch's range.  The linear-time
    kernels are checked against the per-sample-code path instead.  (The no-deformation kernel has no oracle here:
    checks 1 and 3 cover it.)
    Control: a tile holding the values of the tile two iterations earlier on its CTA (a stale buffer), and a tile whose
    rows are shifted by one, each applied to the reference, must exceed these tolerances 10x."""
    kernel, shape, wh = case
    full = _full(case)
    pk = full["packed"]
    rays, taken, idx, sub_info, local = _probe(case)
    n = pk["t_starts"].shape[0]
    print(f"\n{case}: {rays.numel()} probe rays, {idx.numel()} samples; tiles "
          f"{[(lab, t) for lab, t in taken][:12]}{' ...' if len(taken) > 12 else ''}")
    lerp = KERNELS[kernel][1] == "lerp"
    want = _lerp_reference(case, rays, idx, sub_info) if lerp else _oracle(case, rays, idx, local)
    got = {"offsets": pk["offsets"].cpu()[idx], "density": pk["sigma"].cpu()[idx][:, None], "rgb_samples": pk["rgb"].cpu()[idx],
           "weights": pk["weights"].cpu()[idx]}
    gray = {k: full[k].cpu()[rays] for k in ("rgb", "accumulation", "depth", "deformation")}
    worst = {}
    for k in ("offsets", "density", "rgb_samples", "weights"):
        worst[k] = rso.tol_ratio(got[k], want[k], *TOL[k])
        torch.testing.assert_close(got[k], want[k].float(), rtol=TOL[k][0], atol=TOL[k][1], msg=lambda m, k=k: f"{case} {k}: {m}")
    l2 = (gray["rgb"] - want["rgb"].float()).norm(dim=-1)
    worst["rgb L2"] = float(l2.max()) / RGB_L2
    assert l2.max() < RGB_L2, (case, float(l2.max()), rays[l2.argmax()].item())
    for k in ("accumulation", "deformation"):
        worst[k] = rso.tol_ratio(gray[k], want[k], *TOL[k])
        torch.testing.assert_close(gray[k], want[k].float(), rtol=TOL[k][0], atol=TOL[k][1])
    if not lerp:
        mid = ((pk["t_starts"].cpu()[idx] + pk["t_ends"].cpu()[idx]) / 2).double()         # pl.render's float32 steps
        w = want["weights"][:, 0].double()
        acc = torch.zeros(rays.numel(), dtype=torch.float64).index_add_(0, local, w)
        dep = torch.zeros(rays.numel(), dtype=torch.float64).index_add_(0, local, w * mid) / (acc + 1e-10)
        dep = dep.clamp(*full["clip"])
        worst["depth"] = rso.tol_ratio(gray["depth"][:, 0], dep, *TOL["depth"])
        torch.testing.assert_close(gray["depth"][:, 0].double(), dep, rtol=TOL["depth"][0], atol=TOL["depth"][1])
    for k, v in worst.items():
        _report(f"worst {k} / tolerance", v)

    # controls, on the reference: position of each global sample in the probe set
    pos = torch.full((n,), -1, dtype=torch.long); pos[idx] = torch.arange(idx.numel())
    tile = rso.tile_of(0, 2, SMS)                   # its buffer's previous user is tile 0, whose rays are probed
    assert tile in [t for _, t in taken]
    rows = torch.arange(tile * rso.TILE, min((tile + 1) * rso.TILE, n))
    src = (tile - 2 * SMS) * rso.TILE + torch.arange(rows.numel())
    assert (pos[rows] >= 0).all() and (pos[src] >= 0).all()
    for name, from_rows in (("stale buffer", src), ("rows shifted by one", torch.cat([rows[1:], rows[-1:]]))):
        ratio = 0.0
        for k in ("offsets", "density", "rgb_samples"):
            mutated = want[k].clone()
            mutated[pos[rows]] = want[k][pos[from_rows]]
            ratio = max(ratio, rso.tol_ratio(mutated, want[k], *TOL[k]))
        _report(f"control '{name}' on tile {tile} (CTA, it) = {rso.tile_place(tile, SMS)}: rejected by", ratio)
        assert ratio >= 10.0, f"{case}: the tolerances see only {ratio:.2f}x of a {name}"


# ---------------------------------------------------------------------------------------------------------------------
# 3. float64 compositing of every ray
# ---------------------------------------------------------------------------------------------------------------------
def _bound_check(what, got, ref, scale, c):
    """|got - ref| <= c U32 scale + FLT_MIN (exact where the scale is 0); returns the worst ratio."""
    bound = c * so.U32 * scale + so.FLT_MIN
    r = rso.bound_ratio(got, ref, bound)
    assert r <= 1.0, f"{what}: worst error / bound {r:.3g}"
    return r


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_every_ray_against_the_float64_composite(case):
    """The full launch's per-ray outputs and weights against the float64 eval-mode composite (render_scale_oracle.
    composite_eval: nan_to_num, white background, clamp; accumulation; expected depth; the deformation renderer) of
    its own packed sigma / rgb / offsets, within scan_oracle's float32 bound error_constant(n) U32 M.  The clip range
    in the workspace header must be exactly the min / max of the float32 midpoints (t_start + t_end) / 2, as
    composite_ray computes them (nsb_march.cuh).
    Control: the composite of a stale tile buffer or of rows shifted by one, in sigma and rgb, must leave some ray of
    that tile 10x outside the bound (its weights, RGB or accumulation)."""
    full = _full(case)
    pk = {k: v.cpu() for k, v in full["packed"].items()}
    info = full["packed_info"].cpu()
    n = pk["t_starts"].shape[0]
    rng = rso.midpoint_range(pk["t_starts"], pk["t_ends"])
    assert full["clip"] == (rng if rng is not None else (1.0, 1.0)), (full["clip"], rng)
    off = pk.get("offsets")
    ref = rso.composite_eval(info, pk["t_starts"], pk["t_ends"], pk["sigma"], pk["rgb"], off)
    c = so.error_constant(info[:, 1])
    ri = pk["ray_indices"].long()
    worst = {"weights": _bound_check("weights", pk["weights"][:, 0], ref["weights"], ref["weights_scale"], c[ri]),
             "rgb": _bound_check("rgb", full["rgb"].cpu(), ref["rgb"], ref["rgb_scale"], c[:, None]),
             "accumulation": _bound_check("accumulation", full["accumulation"].cpu()[:, 0], ref["accumulation"],
                                          ref["accumulation_scale"], c),
             "depth": _bound_check("depth", full["depth"].cpu()[:, 0], ref["depth"], ref["depth_scale"], c)}
    if off is not None:
        worst["deformation"] = _bound_check("deformation", full["deformation"].cpu(), ref["deformation"],
                                            ref["deformation_scale"], c[:, None])
    print(f"\n{case}: clip range {full['clip']}")
    for k, v in worst.items():
        _report(f"worst {k} error / float32 bound", v)

    # controls: the probe tile (iteration >= 2) whose samples carry the most weight (a tile behind an opaque surface
    # composites to the same colour whatever it holds)
    _, taken, _, _, _ = _probe(case)
    w = pk["weights"][:, 0]
    cand = [t for _, t in taken if rso.tile_place(t, SMS)[1] >= 2]
    tile = max(cand, key=lambda t: float(w[t * rso.TILE:(t + 1) * rso.TILE].sum()))
    rays = torch.unique(ri[tile * rso.TILE:min((tile + 1) * rso.TILE, n)])
    idx, sub_info, _ = rso.subset_samples(info, rays)
    for name, mut in (("stale buffer", lambda v: rso.stale_tile(v, tile, SMS, n)),
                      ("rows shifted by one", lambda v: rso.shift_tile_rows(v, tile, n))):
        bad = rso.composite_eval(sub_info, pk["t_starts"][idx], pk["t_ends"][idx], mut(pk["sigma"])[idx],
                                 mut(pk["rgb"])[idx], None, clip=ref["clip"])
        ratio = max([rso.bound_ratio(bad[k], ref[k][rays], c[rays].reshape(-1, *[1] * (ref[k].dim() - 1)) * so.U32 *
                                     ref[k + "_scale"][rays] + so.FLT_MIN) for k in ("rgb", "accumulation")] +
                    [rso.bound_ratio(bad["weights"], ref["weights"][idx],
                                     c[ri[idx]] * so.U32 * ref["weights_scale"][idx] + so.FLT_MIN)])
        _report(f"control '{name}' on tile {tile} (CTA, it) = {rso.tile_place(tile, SMS)}: rejected by", ratio)
        assert ratio >= 10.0, f"{case}: the bound sees only {ratio:.2f}x of a {name}"


# ---------------------------------------------------------------------------------------------------------------------
# 4. the kernels against each other at full scale; 5. determinism
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("other", ["line", "mma_sync"])
def test_kernels_agree_at_full_scale(other):
    """The timestep-stack kernel against the line-gather kernel and the mma.sync kernel on the benchmark's batch, at
    the config-2 tolerances: three gathers and two deformation MLPs that share little code."""
    a, b = _full(("stack", "A", 32.0)), _full((other, "A", 32.0))
    pa, pb = a["packed"], b["packed"]
    for k in ("t_starts", "t_ends", "ray_indices"):
        assert torch.equal(pa[k], pb[k]), k
    print(f"\nstack vs {other}:")
    for k, g in (("offsets", "offsets"), ("density", "sigma"), ("rgb_samples", "rgb"), ("weights", "weights")):
        _report(f"worst {k} / tolerance", rso.tol_ratio(pb[g], pa[g], *TOL[k]))
        torch.testing.assert_close(pb[g], pa[g], rtol=TOL[k][0], atol=TOL[k][1], msg=lambda m, k=k: f"{other} {k}: {m}")
    l2 = (a["rgb"] - b["rgb"]).norm(dim=-1)
    _report("worst per-ray RGB L2", float(l2.max()), RGB_L2)
    assert l2.max() < RGB_L2
    for k in ("accumulation", "depth", "deformation"):
        _report(f"worst {k} / tolerance", rso.tol_ratio(b[k], a[k], *TOL[k]))
        torch.testing.assert_close(b[k], a[k], rtol=TOL[k][0], atol=TOL[k][1])


def test_benchmark_path_is_deterministic():
    """A second launch of render_kernel_tc<4, true, true> on the benchmark's batch gives the same bits."""
    case = ("stack", "A", 32.0)
    first = _full(case)
    o, d, t, _ = _rays("A")
    again = _outputs(_render(*case, o, d, t))
    for k in PER_RAY:
        assert torch.equal(first[k], again[k]), k
    for k in PACKED:
        assert torch.equal(first["packed"][k], again["packed"][k]), k
    assert first["clip"] == again["clip"]
