"""nsb_render_forward (ops.render_rays): sampler -> field -> composite in one launch (fixed march) / the cooperative
march launch + one fused launch (occupancy grid), without host synchronisation.  The fused path runs the device code of
the stand-alone kernels, so every output must be BIT-IDENTICAL to nsb_march_* + nsb_field_forward + nsb_composite_forward."""
import pytest
import torch

from conftest import native_from_oracle, oracle_params

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TRAINED = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
               deform_last_scale=1e-3)


@pytest.fixture(scope="module")
def trained():
    P = oracle_params(TRAINED)
    return P, native_from_oracle(P, DEV)


@pytest.fixture(scope="module")
def trained_mma(trained):
    """The same parameters with the deformation MLP of the inference kernels on mma.sync (NSB_TCGEN05=0): what the
    training kernels run, and the render kernel render_kernel_ws<true, .>."""
    return trained[0], native_from_oracle(trained[0], DEV, tcgen05=False)


def _rays(R, seed):
    from oracle.gen_golden import ring_rays
    o, d, t, _ = ring_rays(R, seed)
    return o.to(DEV), d.to(DEV), t.to(DEV)


def _same(a, b):
    return a.shape == b.shape and bool(torch.equal(a, b))


@pytest.mark.parametrize("w_hash,w_deform,deform", [(32.0, 7.0, True), (1.5, 3.3, True), (32.0, None, False)])
@pytest.mark.parametrize("R,n_per", [(300, 77), (5, 1), (1, 200)])
def test_fixed_march_one_launch_is_bit_identical_to_the_three_kernel_path(trained, w_hash, w_deform, deform, R, n_per):
    from nersemble_b200 import ops
    P, NP = trained
    o, d, t = _rays(R, 3)
    ts, te, ri, info = ops.march_fixed(o, d, P.aabb, n_per, 0.011, 0.2)
    want = ops.render_packed(NP, o, d, t, ts, te, ri, info, window_hash=w_hash, window_deform=w_deform,
                             use_deformation=deform, training=False)
    got = ops.render_rays(NP, o, d, t, window_hash=w_hash, window_deform=w_deform, use_deformation=deform, sampler="fixed",
                          n_per_ray=n_per, near_plane=0.2, step=0.011)
    for k in ("rgb", "accumulation", "depth") + (("deformation",) if deform else ()):
        assert _same(got[k], want[k]), k
    assert _same(got["packed_info"], info) and _same(got["num_samples_per_ray"], want["num_samples_per_ray"])
    pk = got.packed()
    assert _same(pk["t_starts"], ts) and _same(pk["t_ends"], te) and _same(pk["ray_indices"], ri)
    assert _same(pk["sigma"], want["density"][:, 0]) and _same(pk["rgb"], want["rgb_samples"]) and _same(pk["weights"], want["weights"])
    if deform:
        assert _same(pk["offsets"], want["offsets"])


@pytest.mark.parametrize("mode", ["one_traversal", "one_traversal_mma", "count_scan_fill"])
@pytest.mark.parametrize("levels", [1, 2])
def test_occupancy_march_fused_is_bit_identical(trained, trained_mma, levels, mode):
    from nersemble_b200 import ops
    from oracle.gen_golden import blob_grid
    from oracle.tp import nerfacc_cpu
    P, NP = trained_mma if mode == "one_traversal_mma" else trained       # bit-identity holds within one tensor role
    R = 700                                            # > 256 * ... several scan slabs per CTA chunk is covered by R = 40 000 below
    o, d, t = _rays(R, 11)
    d[5] = torch.tensor([0.0, 0.0, -1.0]); o[5] = torch.tensor([0.1, 0.2, 9.0])
    o[6] = torch.tensor([50.0, 50.0, 50.0]); d[6] = torch.tensor([0.0, 1.0, 0.0])          # misses the box: zero samples
    occ = torch.stack([blob_grid(20 + l) for l in range(levels)]).to(DEV)
    aabbs = torch.stack([nerfacc_cpu._enlarge_aabb(P.aabb.reshape(-1), 2 ** l) for l in range(levels)]).to(DEV)
    gen = torch.Generator().manual_seed(2)
    near = (torch.full((R,), 0.2) + torch.rand((R,), generator=gen) * 0.011).to(DEV)
    far = torch.full((R,), 1e3, device=DEV)
    ts, te, ri, info = ops.march_occupancy(o, d, near, far, occ, aabbs, 0.011, 0.0)
    want = ops.render_packed(NP, o, d, t, ts, te, ri, info, window_hash=32.0, window_deform=7.0, training=False)
    # cooperative march launch, then the fused field + composite launch.  "one_traversal": ONE traversal into per-ray
    # slots + packing copy (the default), wgmma deformation role; "one_traversal_mma": the same on the mma.sync role
    # (render_kernel_ws<true, 2>); "count_scan_fill": the march traverses the grid twice (count | scan | fill)
    got = ops.render_rays(NP, o, d, t, window_hash=32.0, window_deform=7.0, sampler="occupancy", near_planes=near,
                          far_planes=far, binaries=occ, aabbs=aabbs, step=0.011, single_traversal=mode != "count_scan_fill")
    assert _same(got["packed_info"], info)
    for k in ("rgb", "accumulation", "depth", "deformation"):
        assert _same(got[k], want[k]), k
    pk = got.packed()
    assert pk["t_starts"].shape[0] == ts.shape[0] > 1000
    assert _same(pk["t_starts"], ts) and _same(pk["t_ends"], te) and _same(pk["ray_indices"], ri)
    assert _same(pk["sigma"], want["density"][:, 0]) and _same(pk["weights"], want["weights"])


def test_occupancy_scan_over_many_rays_and_capacity_overflow(trained):
    """40 000 rays: every CTA of the cooperative march scans several slabs; then a too-small capacity must raise the
    status flag (and never write out of bounds) instead of corrupting memory."""
    from nersemble_b200 import ops
    from oracle.gen_golden import blob_grid
    P, NP = trained
    R = 40000
    o, d, t = _rays(R, 5)
    occ = blob_grid(7)[None].to(DEV)
    aabbs = P.aabb.reshape(1, 6).to(DEV)
    near = torch.full((R,), 0.2, device=DEV); far = torch.full((R,), 1e3, device=DEV)
    ts, te, ri, info = ops.march_occupancy(o, d, near, far, occ, aabbs, 0.011, 0.0)
    got = ops.render_rays(NP, o, d, t, window_hash=32.0, window_deform=7.0, sampler="occupancy", near_planes=near,
                          far_planes=far, binaries=occ, aabbs=aabbs, step=0.011)
    assert _same(got["packed_info"], info)
    want = ops.render_packed(NP, o, d, t, ts, te, ri, info, window_hash=32.0, window_deform=7.0, training=False)
    assert _same(got["rgb"], want["rgb"]) and _same(got["depth"], want["depth"])
    n = int(ts.shape[0])
    small = ops.render_rays(NP, o, d, t, window_hash=32.0, window_deform=7.0, sampler="occupancy", near_planes=near,
                            far_planes=far, binaries=occ, aabbs=aabbs, step=0.011, capacity=n // 2)
    torch.cuda.synchronize()
    hdr = small["_buffers"]["header"]
    assert (int(hdr[1]) >> 32) == 1 and int(hdr[2]) <= n // 2      # status raised, the kept samples fit the workspace
    with pytest.raises(RuntimeError):
        small.packed()


@pytest.mark.parametrize("tensor_role", ["mma.sync", "tcgen05"])
def test_plugin_eval_paths_use_the_fused_render(trained, monkeypatch, tensor_role):
    """NeRSembleNGPModel eval: get_outputs_for_camera_ray_bundle (no host sync) and get_outputs (full contract) agree bit
    for bit with the training-path kernels run in eval mode when both run the mma.sync deformation role; with the
    wgmma role (flag name "tcgen05", the default of the fused render) they agree to fp16-operand rounding."""
    from nersemble_b200 import ops
    from nersemble_b200.nerfstudio_shim import RayBundle
    monkeypatch.setattr(ops, "USE_TCGEN05", tensor_role == "tcgen05")
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P, _ = trained
    m = make_model(T=4, log2T=14, eval_num_rays_per_chunk=500)
    load_oracle_params_into(m, P)
    m = m.to(DEV).eval()
    m.sched_window_hash_encodings.value = 32.0; m.sched_window_deform.value = 7.0
    m.occupancy_grid.binaries[0] = blob_grid(5).to(DEV)
    H, W = 30, 40
    o, d, t = _rays(H * W, 9)
    rb = RayBundle(origins=o.view(H, W, 3), directions=d.view(H, W, 3), pixel_area=torch.ones(H, W, 1, device=DEV),
                   camera_indices=torch.zeros(H, W, 1, dtype=torch.long, device=DEV), times=t.view(H, W, 1))
    with torch.no_grad():
        img = m.get_outputs_for_camera_ray_bundle(rb)
        m.use_fused_render = False
        ref = m.get_outputs_for_camera_ray_bundle(rb)
        m.use_fused_render = True
        flat = RayBundle(origins=o, directions=d, pixel_area=torch.ones(H * W, 1, device=DEV),
                         camera_indices=torch.zeros(H * W, 1, dtype=torch.long, device=DEV), times=t)
        full = m.get_outputs(flat)
        m.use_fused_render = False
        full_ref = m.get_outputs(flat)
    rs, rs_ref = full["ray_samples"][0], full_ref["ray_samples"][0]
    assert _same(full["ray_indices"][0], full_ref["ray_indices"][0]) and _same(rs.frustums.starts, rs_ref.frustums.starts)
    assert _same(rs.frustums.origins, rs_ref.frustums.origins) and _same(rs.times, rs_ref.times)
    assert _same(img["num_samples_per_ray"], ref["num_samples_per_ray"]) and _same(full["num_samples_per_ray"], full_ref["num_samples_per_ray"])
    if tensor_role == "mma.sync":
        for k in ("rgb", "accumulation", "depth", "deformation"):
            assert _same(img[k], ref[k]), k
            assert _same(full[k], full_ref[k]), k
        assert _same(full["weights"][0], full_ref["weights"][0]) and _same(rs.frustums.offsets, rs_ref.frustums.offsets)
    else:
        for a, b in ((img, ref), (full, full_ref)):
            assert (a["rgb"] - b["rgb"]).norm(dim=-1).max() < 1e-3
            torch.testing.assert_close(a["accumulation"], b["accumulation"], rtol=0, atol=1e-3)
            torch.testing.assert_close(a["depth"], b["depth"], rtol=1e-3, atol=1e-3)
            torch.testing.assert_close(a["deformation"], b["deformation"], rtol=5e-3, atol=1e-5)
        torch.testing.assert_close(full["weights"][0], full_ref["weights"][0], rtol=5e-3, atol=2e-5)
        torch.testing.assert_close(rs.frustums.offsets, rs_ref.frustums.offsets, rtol=2e-3, atol=3e-6)


def test_sync_free_training_sampler_matches_the_four_sync_path(trained):
    """Training-mode get_outputs: cooperative march + density pre-pass with a device-side count + visibility/packing in
    one launch (one host sync) against the original path (march count / cumsum / fill, occs.mean().item(), density_fn,
    visibility kernel, boolean indexing): the same kept samples bit for bit, the same outputs and gradients."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P, _ = trained
    m = make_model(T=4, log2T=14)
    load_oracle_params_into(m, P)
    m = m.to(DEV).train()
    m.sched_window_hash_encodings.value = 32.0; m.sched_window_deform.value = 7.0
    occ = blob_grid(5)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(DEV))
    R = 900
    o, d, t = _rays(R, 13)
    o[6] = torch.tensor([50.0, 50.0, 50.0], device=DEV); d[6] = torch.tensor([0.0, 1.0, 0.0], device=DEV)
    rb = RayBundle(origins=o, directions=d, pixel_area=torch.ones(R, 1, device=DEV),
                   camera_indices=torch.zeros(R, 1, dtype=torch.long, device=DEV), times=t[:, None] if t.dim() == 1 else t)
    jit = torch.rand(R, generator=torch.Generator().manual_seed(1)).to(DEV)
    res = {}
    for fused in (True, False, "no_reuse"):
        m.use_fused_sampler = bool(fused)
        m.prepass_reuse = fused is True          # True: the differentiable forward takes the pre-pass's packed features
        m.zero_grad(set_to_none=True)
        m.field.hash_ensemble.pending_table_grad = None
        out = m.get_outputs(rb, jitter=jit)
        (out["rgb"].sum() + out["accumulation"].sum() * 0.3).backward()
        res[fused] = (out, m.field.mlp_base.params.grad.clone(), m.time_embedding.weight.grad.clone())
    a, b = res[True][0], res[False][0]
    assert a["ray_indices"][0].numel() > 2000
    assert _same(a["ray_indices"][0], b["ray_indices"][0])
    assert _same(a["ray_samples"][0].frustums.starts, b["ray_samples"][0].frustums.starts)
    assert _same(a["ray_samples"][0].frustums.ends, b["ray_samples"][0].frustums.ends)
    assert _same(a["num_samples_per_ray"], b["num_samples_per_ray"])
    for k in ("rgb", "accumulation", "depth", "deformation"):
        assert _same(a[k], b[k]), k
    assert _same(a["weights"][0], b["weights"][0])
    # gradients: float atomics in the scatter -> rounding-order noise only
    torch.testing.assert_close(res[True][1], res[False][1], rtol=1e-3, atol=1e-6)
    torch.testing.assert_close(res[True][2], res[False][2], rtol=1e-3, atol=1e-7)
    c = res["no_reuse"][0]          # pre-pass reuse on/off: the same features, so the same forward bit for bit
    for k in ("rgb", "accumulation", "depth", "deformation"):
        assert _same(a[k], c[k]), k
    assert _same(a["weights"][0], c["weights"][0])
    torch.testing.assert_close(res[True][1], res["no_reuse"][1], rtol=1e-3, atol=1e-6)
    torch.testing.assert_close(res[True][2], res["no_reuse"][2], rtol=1e-3, atol=1e-7)
    # an empty occupancy grid: the zero-sample guard (one fake sample on ray 0) on both paths
    m.occupancy_grid.binaries[:] = False
    with torch.no_grad():
        m.use_fused_sampler = True
        z1 = m.get_outputs(rb, jitter=jit)
        m.use_fused_sampler = False
        z0 = m.get_outputs(rb, jitter=jit)
    assert z1["ray_indices"][0].numel() == 1 and _same(z1["rgb"], z0["rgb"]) and _same(z1["depth"], z0["depth"])
    assert _same(z1["num_samples_per_ray"], z0["num_samples_per_ray"])


def test_visibility_compact_moves_payload_rows_with_their_samples():
    from nersemble_b200 import ops
    g = torch.Generator().manual_seed(4)
    R = 300
    cnt = torch.randint(0, 90, (R,), generator=g); cnt[7] = 0; cnt[R - 1] = 0
    n = int(cnt.sum()); cap = n + 100
    ri = torch.repeat_interleave(torch.arange(R), cnt)
    ts = torch.rand((n,), generator=g); te = ts + 0.011
    sig = torch.rand((n,), generator=g) * 60
    pad = lambda x, fill=0: torch.cat([x, torch.full((cap - n,) + tuple(x.shape[1:]), fill, dtype=x.dtype)])
    info = torch.stack([cnt.cumsum(0) - cnt, cnt], -1)
    cand = {"t_starts": pad(ts).to(DEV), "t_ends": pad(te).to(DEV), "ray_indices": pad(ri.int()).to(DEV),
            "packed_info": info.to(DEV), "capacity": cap}
    payload = {"feat": torch.randn((cap, 32), generator=g).half().to(DEV), "xs": torch.rand((cap, 4), generator=g).to(DEV),
               "corner_vals": torch.randn((cap, 16, 8, 2), generator=g).half().to(DEV)}
    occs_mean = torch.tensor(0.3, device=DEV)
    mask, kept = ops.visibility_mask(info.to(DEV), ts.to(DEV), te.to(DEV), sig.to(DEV), 1e-3, min(0.5, 0.3))
    got = ops.visibility_compact(cand, pad(sig).to(DEV), 1e-3, 0.5, alpha_thre_cap=occs_mean, payload=payload)
    k = int(got["n_total"].item())
    assert k == int(mask.sum()) and 0 < k < n
    assert _same(got["packed_info"][:, 1], kept.long())
    assert _same(got["t_starts"][:k], ts.to(DEV)[mask]) and _same(got["ray_indices"][:k], ri.int().to(DEV)[mask])
    for name in ("feat", "xs", "corner_vals"):
        assert _same(got[name][:k], payload[name][:n][mask]), name


def test_plugin_camera_frame_uses_the_frame_table(trained):
    """A camera frame carries ONE timestep: get_outputs_for_camera_ray_bundle hoists the member blend into a per-frame
    table (NeRSembleNGPModel.frame_tables).  Same image as the per-sample blend within the north-star tolerance; the
    cached table follows the timestep and the table values (in-place optimiser updates bump the version)."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid
    from test_plugin_cpu import make_model
    from test_plugin_gpu import load_oracle_params_into
    P, _ = trained
    m = make_model(T=4, log2T=14, eval_num_rays_per_chunk=700)
    load_oracle_params_into(m, P)
    m = m.to(DEV).eval()
    m.frame_table_min_rays = 1
    m.sched_window_hash_encodings.value = 32.0; m.sched_window_deform.value = 7.0
    m.occupancy_grid.binaries[0] = blob_grid(5).to(DEV)
    H, W = 30, 40
    o, d, _ = _rays(H * W, 9)
    imgs = {}
    with torch.no_grad():
        for tv in (1.0 / 3.0, 1.0):
            rb = RayBundle(origins=o.view(H, W, 3), directions=d.view(H, W, 3), pixel_area=torch.ones(H, W, 1, device=DEV),
                           camera_indices=torch.zeros(H, W, 1, dtype=torch.long, device=DEV),
                           times=torch.full((H, W, 1), tv, device=DEV))
            m.frame_tables = True
            a = m.get_outputs_for_camera_ray_bundle(rb)
            assert m.native_params()._frame[0][0] == round(tv * 3)          # the cached table is this frame's timestep
            m.frame_tables = False
            b = m.get_outputs_for_camera_ray_bundle(rb)
            assert _same(a["num_samples_per_ray"], b["num_samples_per_ray"])
            torch.testing.assert_close(a["deformation"], b["deformation"], rtol=5e-3, atol=1e-6)    # weights differ by rounding
            assert (a["rgb"] - b["rgb"]).norm(dim=-1).max() < 1e-3
            torch.testing.assert_close(a["accumulation"], b["accumulation"], rtol=0, atol=1e-3)
            torch.testing.assert_close(a["depth"], b["depth"], rtol=1e-3, atol=1e-3)
            imgs[tv] = a["rgb"]
        assert (imgs[1.0] - imgs[1.0 / 3.0]).abs().max() > 1e-3              # the two timesteps differ
        # the tables change in place (an optimiser step): the cached frame table must not be reused
        m.frame_tables = True
        m.field.hash_ensemble.tables.mul_(0.5)
        c = m.get_outputs_for_camera_ray_bundle(rb)["rgb"]
        m.frame_tables = False
        e = m.get_outputs_for_camera_ray_bundle(rb)["rgb"]
        assert (c - e).norm(dim=-1).max() < 1e-3 and (c - imgs[1.0]).abs().max() > 1e-3
