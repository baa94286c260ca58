"""Plugin surface on the GPU: NeRSembleNGPModel.get_outputs (sampler + fused field + composite) against the goldens
produced by the REAL reference model, plus the component modules."""
import pytest
import torch

from conftest import load_golden, oracle_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision
from test_plugin_cpu import make_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def load_oracle_params_into(model, P):
    from nersemble_b200 import packing
    with torch.no_grad():
        model.field.hash_ensemble.load_tcnn_grids(packing.tables_to_tcnn(P.tables))
        model.field.mlp_base.params.copy_(torch.cat([w.reshape(-1) for w in P.base_w]))
        model.field.mlp_head.params.copy_(torch.cat([w.reshape(-1) for w in P.head_w]))
        se3 = model.deformation_field.se3_field
        for i, layer in enumerate(se3.mlp_stem.layers):
            layer.weight.copy_(P.deform_w[i]); layer.bias.copy_(P.deform_b[i])
        se3.mlp_r.layers[0].weight.copy_(P.r_w); se3.mlp_r.layers[0].bias.copy_(P.r_b)
        se3.mlp_v.layers[0].weight.copy_(P.v_w); se3.mlp_v.layers[0].bias.copy_(P.v_b)
        model.time_embedding.weight.copy_(P.time_emb)
        model.time_embedding_deformation.weight.copy_(P.time_emb_deform)


def _bundle(g):
    from nersemble_b200.nerfstudio_shim import RayBundle
    R = g["origins"].shape[0]
    return RayBundle(origins=g["origins"].to(DEV), directions=g["directions"].to(DEV), pixel_area=torch.ones(R, 1, device=DEV),
                     camera_indices=g["camera_indices"].to(DEV), times=g["times"].to(DEV))


@pytest.mark.parametrize("name", ["occ_eval_soft", "occ_eval_whash1", "occ_train_prepass"])
def test_model_get_outputs_vs_reference_golden(name):
    from oracle.gen_golden import blob_grid
    g, meta = load_golden(name)
    P = oracle_params(meta["knobs"])
    m = make_model(T=meta["knobs"]["n_timesteps"], log2T=meta["knobs"]["log2_hashmap_size"])
    load_oracle_params_into(m, P)
    m = m.to(DEV)
    m.sched_window_hash_encodings.value = meta["w_hash"]
    m.sched_window_deform.value = meta["w_deform"]
    occ = blob_grid(meta["grid_seed"])
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(DEV))
    m.train(meta["training"])
    jitter = None
    if meta["training"]:
        torch.manual_seed(meta["jitter_seed"])
        jitter = torch.rand(meta["R"]).to(DEV)
    with torch.no_grad():
        out = m.get_outputs(_bundle(g), jitter=jitter)
    rs = out["ray_samples"][0]
    ri = out["ray_indices"][0].cpu()
    if not meta["training"]:
        # eval: no pre-pass -> the marcher alone decides; bit-exact to nerfacc semantics
        assert torch.equal(ri, g["ray_indices"])
        assert torch.equal(rs.frustums.starts[:, 0].cpu(), g["t_starts"]) and torch.equal(rs.frustums.ends[:, 0].cpu(), g["t_ends"])
        torch.testing.assert_close(rs.frustums.offsets.cpu(), g["offsets"], rtol=5e-3, atol=5e-6)
        torch.testing.assert_close(out["weights"][0].cpu(), g["weights"], rtol=2e-2, atol=1e-4)
    else:
        # training: the visibility pre-pass thresholds fp16-path densities; allow a handful of flips
        assert abs(ri.numel() - g["ray_indices"].numel()) <= max(4, g["ray_indices"].numel() // 200)
    assert (out["rgb"].cpu() - g["rgb"]).norm(dim=-1).max() < 1e-3
    torch.testing.assert_close(out["accumulation"].cpu(), g["accumulation"], rtol=0, atol=2e-3)
    torch.testing.assert_close(out["depth"].cpu(), g["depth"], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(out["deformation"].cpu(), g["deformation"], rtol=2e-2, atol=2e-5)
    assert out["num_samples_per_ray"].sum().item() == ri.numel()


def test_field_density_fn_and_components():
    g, meta = load_golden("density_fn_kernel")
    P = oracle_params(meta["knobs"])
    m = make_model(T=4, log2T=14)
    load_oracle_params_into(m, P)
    m = m.to(DEV).eval()
    m.sched_window_hash_encodings.value = meta["w_hash"]
    m.sched_window_deform.value = meta["w_deform"]
    with torch.no_grad():
        sig = m.field_density_fn(g["positions"].to(DEV), g["times"].to(DEV)).cpu()
    torch.testing.assert_close(sig, g["density"], rtol=5e-3, atol=1e-5)
    # component modules: HashEnsemble.forward and SE3DeformationField.compute_offsets vs the oracle
    Precision.mode = "kernel"
    gen = torch.Generator().manual_seed(3)
    x = torch.rand((300, 3), generator=gen)
    code = torch.randn((300, 32), generator=gen) * 0.2
    with torch.no_grad():
        want = pl.hash_ensemble(P, x, code, 20.25)
        got = m.field.hash_ensemble(x.to(DEV), code.to(DEV), window_hash_encodings=20.25).float().cpu()
    assert got.dtype == torch.float32 and ((got - want).abs().max() / want.abs().max()) < 3e-3
    pos = P.aabb[0] + torch.rand((300, 3), generator=gen) * (P.aabb[1] - P.aabb[0])
    wc = P.time_emb_deform[torch.randint(0, 4, (300,), generator=gen)]
    with torch.no_grad():
        want_o = pl.compute_offsets(P, pos, wc, 5.5)
        got_o = m.deformation_field.compute_offsets(pos.to(DEV), wc.to(DEV), 5.5).cpu()
    torch.testing.assert_close(got_o, want_o, rtol=5e-3, atol=5e-6)
    # Field component API (fields/nersemble_nerfacto_field.py:228-248): density_fn with explicit time codes = the
    # oracle's field_density on the same positions
    tsteps = torch.randint(0, 4, (300,), generator=gen)
    with torch.no_grad():
        want_s, _ = pl.field_density(P, pos, P.time_emb[tsteps], 20.25)
        got_s = m.field.density_fn(pos.to(DEV), times=None, window_hash_encodings=20.25,
                                   time_codes=P.time_emb[tsteps].to(DEV)).cpu()
    torch.testing.assert_close(got_s.reshape(-1), want_s.reshape(-1), rtol=5e-3, atol=1e-5)
    Precision.mode = "reference"


def test_occupancy_update_and_full_frame_render():
    """update_every_n_steps through the fused density kernel, then a small full-frame render in chunks."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    P = oracle_params(dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
                           deform_last_scale=1e-3))
    m = make_model(T=4, log2T=14, eval_num_rays_per_chunk=1000)
    load_oracle_params_into(m, P)
    m = m.to(DEV).train()
    cb = m.get_training_callbacks(None)[0]
    torch.manual_seed(0)
    cb.run_callback(0)                                    # warm-up step: all 128^3 cells evaluated
    frac = m.occupancy_grid.binaries.float().mean().item()
    assert 0.0 < frac < 1.0 and m.occupancy_grid.occs.max() > 0
    cb.run_callback(256 * 16)                             # post-warm-up path (uniform + occupied cells)
    m.eval()
    H, W = 24, 40
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1.5, 1.5, W), indexing="ij")
    o = torch.tensor([0.0, 0.0, 9.0]).expand(H, W, 3)
    d = torch.stack([xs, ys, torch.full_like(xs, -9.0)], -1); d = d / d.norm(dim=-1, keepdim=True)
    rb = RayBundle(origins=o.contiguous().to(DEV), directions=d.to(DEV), pixel_area=torch.ones(H, W, 1, device=DEV),
                   camera_indices=torch.zeros(H, W, 1, dtype=torch.long, device=DEV), times=torch.full((H, W, 1), 0.34, device=DEV))
    m.frame_table_min_rays = 1
    img_frame = m.get_outputs_for_camera_ray_bundle(rb)      # one timestep for the frame: per-frame blended table
    m.frame_tables = False
    img = m.get_outputs_for_camera_ray_bundle(rb)            # per-sample member blend
    assert (img_frame["rgb"] - img["rgb"]).norm(dim=-1).max() < 1e-3 and torch.equal(img_frame["num_samples_per_ray"], img["num_samples_per_ray"])
    assert img["rgb"].shape == (H, W, 3) and img["depth"].shape == (H, W, 1) and torch.isfinite(img["rgb"]).all()
    assert img["rgb"].min() >= 0 and img["rgb"].max() <= 1
    flat = RayBundle(origins=rb.origins.view(-1, 3), directions=rb.directions.view(-1, 3),
                     pixel_area=rb.pixel_area.view(-1, 1), camera_indices=rb.camera_indices.view(-1, 1),
                     times=rb.times.view(-1, 1))
    assert m.get_outputs(flat)["rgb"].grad_fn is None   # eval mode is inference-only, even with autograd enabled
    with torch.no_grad():
        full = m.get_outputs(flat)
    torch.testing.assert_close(img["rgb"].view(-1, 3), full["rgb"], rtol=0, atol=1e-6)   # chunking is exact


def test_training_step_gradients_and_descent():
    """use_deformation_field=False recipe: end-to-end gradients through the plugin model (sampler -> fused field ->
    composite -> losses) vs autograd through the oracle, then a few Adam steps must reduce the loss."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid, ring_rays
    from oracle.tp import nerfacc_cpu
    Precision.mode = "kernel"
    knobs = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0, deform_last_scale=1e-3)
    P = pl.random_params(**knobs)
    m = make_model(T=4, log2T=14, use_deformation_field=False, window_deform_end=0,
                   lambda_near_loss=0, lambda_empty_loss=0, lambda_depth_loss=0, lambda_dist_loss=1e-2, lambda_alpha_loss=1e-2)
    with torch.no_grad():
        from nersemble_b200 import packing
        m.field.hash_ensemble.load_tcnn_grids(packing.tables_to_tcnn(P.tables))
        m.field.mlp_base.params.copy_(torch.cat([w.reshape(-1) for w in P.base_w]))
        m.field.mlp_head.params.copy_(torch.cat([w.reshape(-1) for w in P.head_w]))
        m.time_embedding.weight.copy_(P.time_emb)
    m = m.to(DEV).train()
    m.sched_window_hash_encodings.value = 32.0
    occ = blob_grid(3)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(DEV))
    R = 64
    o, d, times, cams = ring_rays(R, 21)
    gen = torch.Generator().manual_seed(1)
    batch = {"image": torch.rand((R, 3), generator=gen), "alpha_map": torch.randint(0, 256, (R, 1), generator=gen).float()}
    rb = RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV),
                   camera_indices=cams.to(DEV), times=times.to(DEV))
    m.sampler.eval()          # no stratified jitter / pre-pass: same samples as the oracle marcher
    out = m.get_outputs(rb)
    ld = m.get_loss_dict(out, batch)
    loss = sum(ld.values())
    loss.backward()
    # ---- oracle: same samples, same losses, autograd
    ts, te, ri = pl.sample_occupancy(P, o, d, times, occ[None], 0.0, 0.011, 0.2, 1e3, 1e-2, 0.0, training=False)
    assert torch.equal(ri, out["ray_indices"][0].cpu())
    P.requires_grad_(True)
    tsteps = pl.timesteps_from_times(times[ri], 4)
    pos = o[ri] + d[ri] * ((ts + te)[:, None] / 2)
    sigma, geo = pl.field_density(P, pos, P.time_emb[tsteps], 32.0)
    rgb_s = pl.field_rgb(P, d[ri], geo)
    info = nerfacc_cpu.pack_info(ri, R)
    w = nerfacc_cpu.render_weight_from_density(ts, te, sigma[:, 0], info)[0]
    acc = nerfacc_cpu.accumulate_along_rays(w, None, ri, R)
    comp = nerfacc_cpu.accumulate_along_rays(w, rgb_s, ri, R) + (1.0 - acc)
    mid = (ts + te)[:, None] / 2
    depth = torch.clip(nerfacc_cpu.accumulate_along_rays(w, mid, ri, R) / (acc + 1e-10), mid.min(), mid.max())
    o_ld = pl.loss_dict({"rgb": comp, "accumulation": acc, "depth": depth, "weights": w[:, None]}, ts, te, ri, batch,
                        eps_depth=0.5, lam_alpha=1e-2, lam_near=0, lam_empty=0, lam_depth=0, lam_dist=1e-2)
    o_loss = sum(o_ld.values())
    o_loss.backward()
    assert abs(loss.item() - o_loss.item()) < 2e-3 * abs(o_loss.item()) + 1e-5
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(m.field.mlp_head.params.grad.cpu(), torch.cat([x.grad.reshape(-1) for x in P.head_w])) < 3e-2
    assert rel(m.field.mlp_base.params.grad.cpu(), torch.cat([x.grad.reshape(-1) for x in P.base_w])) < 3e-2
    assert rel(m.time_embedding.weight.grad.cpu(), P.time_emb.grad) < 3e-2
    got_t = m.field.hash_ensemble.tables.grad.cpu()
    cos = torch.nn.functional.cosine_similarity(got_t.reshape(1, -1), P.tables.grad.reshape(1, -1)).item()
    assert cos > 0.999, cos
    # ---- a few optimiser steps on the same batch reduce the loss
    groups = m.get_param_groups()
    opt = torch.optim.Adam([{"params": groups["fields"], "lr": 5e-3}, {"params": groups["embeddings"], "lr": 5e-3}], eps=1e-15)
    first = loss.item()
    for _ in range(20):
        opt.zero_grad(set_to_none=True)
        out = m.get_outputs(rb)
        l = sum(m.get_loss_dict(out, batch).values())
        l.backward()
        opt.step()
    assert l.item() < 0.85 * first, (first, l.item())
    Precision.mode = "reference"


def test_full_recipe_training_step_gradients():
    """The full recipe (deformation field + hash ensemble): end-to-end parameter gradients through the plugin model vs
    autograd through the oracle, then Adam steps over all three parameter groups reduce the loss."""
    from nersemble_b200 import packing
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid, ring_rays
    from oracle.tp import nerfacc_cpu
    Precision.mode = "kernel"
    knobs = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0, deform_last_scale=0.02)
    P = pl.random_params(**knobs)
    m = make_model(T=4, log2T=14, lambda_near_loss=0, lambda_empty_loss=0, lambda_depth_loss=0, lambda_dist_loss=1e-2,
                   lambda_alpha_loss=1e-2)
    load_oracle_params_into(m, P)
    m = m.to(DEV).train()
    m.sched_window_hash_encodings.value = 32.0
    m.sched_window_deform.value = 5.5
    occ = blob_grid(3)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    R = 64
    o, d, times, cams = ring_rays(R, 21)
    gen = torch.Generator().manual_seed(1)
    batch = {"image": torch.rand((R, 3), generator=gen), "alpha_map": torch.randint(0, 256, (R, 1), generator=gen).float()}
    rb = RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV),
                   camera_indices=cams.to(DEV), times=times.to(DEV))
    m.sampler.eval()
    out = m.get_outputs(rb)
    assert "deformation" in out and out["ray_samples"][0].frustums.offsets is not None
    loss = sum(m.get_loss_dict(out, batch).values())
    loss.backward()
    # ---- oracle
    ts, te, ri = pl.sample_occupancy(P, o, d, times, occ[None], 0.0, 0.011, 0.2, 1e3, 1e-2, 0.0, training=False)
    assert torch.equal(ri, out["ray_indices"][0].cpu())
    P.requires_grad_(True)
    r = pl.render(P, o, d, times, ts, te, ri, window_hash=32.0, window_deform=5.5, training=True)
    o_ld = pl.loss_dict(r, ts, te, ri, batch, eps_depth=0.5, lam_alpha=1e-2, lam_near=0, lam_empty=0, lam_depth=0, lam_dist=1e-2)
    o_loss = sum(o_ld.values())
    o_loss.backward()
    assert abs(loss.item() - o_loss.item()) < 3e-3 * abs(o_loss.item()) + 1e-5
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    se3 = m.deformation_field.se3_field
    for l, layer in enumerate(se3.mlp_stem.layers):
        assert rel(layer.weight.grad.cpu(), P.deform_w[l].grad) < 6e-2, l
        assert rel(layer.bias.grad.cpu(), P.deform_b[l].grad) < 6e-2, l
    assert rel(se3.mlp_r.layers[0].weight.grad.cpu(), P.r_w.grad) < 5e-2
    assert rel(se3.mlp_v.layers[0].weight.grad.cpu(), P.v_w.grad) < 5e-2
    assert rel(m.time_embedding_deformation.weight.grad.cpu(), P.time_emb_deform.grad) < 6e-2
    assert rel(m.time_embedding.weight.grad.cpu(), P.time_emb.grad) < 4e-2
    assert rel(m.field.mlp_head.params.grad.cpu(), torch.cat([x.grad.reshape(-1) for x in P.head_w])) < 4e-2
    got_t = m.field.hash_ensemble.tables.grad.cpu()
    assert torch.nn.functional.cosine_similarity(got_t.reshape(1, -1), P.tables.grad.reshape(1, -1)).item() > 0.999
    # ---- optimiser steps over the reference's three parameter groups (train_nersemble.py:243-256)
    groups = m.get_param_groups()
    opt = torch.optim.Adam([{"params": groups["fields"], "lr": 5e-3}, {"params": groups["embeddings"], "lr": 5e-3},
                            {"params": [p for p in groups["deformation_field"] if p.requires_grad], "lr": 1e-3}], eps=1e-15)
    first = loss.item()
    for _ in range(20):
        opt.zero_grad(set_to_none=True)
        out = m.get_outputs(rb)
        l = sum(m.get_loss_dict(out, batch).values())
        l.backward()
        opt.step()
    assert l.item() < 0.85 * first, (first, l.item())
    Precision.mode = "reference"


def test_loss_curve_agrees_with_oracle_for_first_steps():
    """SURVEY 8(d) config 3: the first optimiser steps of the CUDA training path follow the oracle's loss curve
    (same parameters, rays, losses and Adam hyper-parameters; oracle = autograd through oracle/pipeline.py on CPU)."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid, ring_rays
    Precision.mode = "kernel"
    knobs = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=12, table_scale=0.5, time_std_scale=100.0, deform_last_scale=0.02)
    P = pl.random_params(**knobs)
    m = make_model(T=4, log2T=12, lambda_near_loss=0, lambda_empty_loss=0, lambda_depth_loss=0, lambda_dist_loss=1e-2,
                   lambda_alpha_loss=1e-2)
    load_oracle_params_into(m, P)
    m = m.to(DEV).train()
    m.sched_window_hash_encodings.value = 32.0
    m.sched_window_deform.value = 5.5
    occ = blob_grid(3)
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.sampler.eval()
    R = 48
    o, d, times, cams = ring_rays(R, 33)
    gen = torch.Generator().manual_seed(2)
    batch = {"image": torch.rand((R, 3), generator=gen), "alpha_map": torch.randint(0, 256, (R, 1), generator=gen).float()}
    rb = RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV),
                   camera_indices=cams.to(DEV), times=times.to(DEV))
    groups = m.get_param_groups()
    opt = torch.optim.Adam([{"params": groups["fields"], "lr": 5e-3}, {"params": groups["embeddings"], "lr": 5e-3},
                            {"params": [p for p in groups["deformation_field"] if p.requires_grad], "lr": 1e-3}], eps=1e-15)
    P.requires_grad_(True)
    o_opt = torch.optim.Adam([{"params": [P.tables] + P.base_w + P.head_w, "lr": 5e-3},
                              {"params": [P.time_emb, P.time_emb_deform], "lr": 5e-3},
                              {"params": P.deform_w + P.deform_b + [P.r_w, P.r_b, P.v_w, P.v_b], "lr": 1e-3}], eps=1e-15)
    ts, te, ri = pl.sample_occupancy(P, o, d, times, occ[None], 0.0, 0.011, 0.2, 1e3, 1e-2, 0.0, training=False)
    got, want = [], []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        l = sum(m.get_loss_dict(m.get_outputs(rb), batch).values())
        l.backward(); opt.step(); got.append(l.item())
        o_opt.zero_grad(set_to_none=True)
        r = pl.render(P, o, d, times, ts, te, ri, window_hash=32.0, window_deform=5.5, training=True)
        ol = sum(pl.loss_dict(r, ts, te, ri, batch, eps_depth=0.5, lam_alpha=1e-2, lam_near=0, lam_empty=0, lam_depth=0,
                              lam_dist=1e-2).values())
        ol.backward(); o_opt.step(); want.append(ol.item())
    assert want[-1] < want[0]
    for a, b in zip(got, want):
        assert abs(a - b) < 2e-2 * abs(b), (got, want)
    Precision.mode = "reference"


def test_training_step_gradients_vs_reference_glue_golden():
    """CUDA backward (all kernels, fused losses, full recipe) against gradients computed by torch autograd through the
    UNMODIFIED reference glue (golden `grads_train`, fp32 'none' precision): same samples, six losses, every parameter.
    Tolerances = fp16 operands / deltas of the kernels (the oracle itself agrees with this golden to 2e-3 on the field side
    and 2e-2 on the deformation side, tests/test_oracle_golden.py)."""
    from nersemble_b200.nerfstudio_shim import RayBundle
    from oracle.gen_golden import blob_grid
    g, meta = load_golden("grads_train")
    P = pl.random_params(**meta["knobs"])
    m = make_model(T=4, log2T=meta["knobs"]["log2_hashmap_size"])          # the script's default lambdas: all six losses
    load_oracle_params_into(m, P)
    m = m.to(DEV).train()
    m.sched_window_hash_encodings.value = meta["w_hash"]
    m.sched_window_deform.value = meta["w_deform"]
    m.sched_eps_depth.value = meta["eps_depth"]
    occ = blob_grid(meta["grid_seed"])
    m.occupancy_grid.binaries[0] = occ.to(DEV)
    m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(DEV))
    m.sampler.eval()
    R = g["origins"].shape[0]
    rb = RayBundle(origins=g["origins"].to(DEV), directions=g["directions"].to(DEV), pixel_area=torch.ones(R, 1, device=DEV),
                   camera_indices=g["camera_indices"].to(DEV), times=g["times"].to(DEV))
    batch = {k[len("batch_"):]: v for k, v in g.items() if k.startswith("batch_")}
    out = m.get_outputs(rb)
    assert torch.equal(out["ray_indices"][0].cpu(), g["ray_indices"])
    ld = m.get_loss_dict(out, batch)
    want_l = {k[len("loss_"):]: v for k, v in g.items() if k.startswith("loss_")}
    assert set(ld) == set(want_l)
    for k in want_l:
        assert abs(ld[k].item() - want_l[k].item()) < 5e-3 * abs(want_l[k].item()) + 1e-8, (k, ld[k].item(), want_l[k].item())
    sum(ld.values()).backward()

    def check(got, want, what, tol, min_cos=0.995):
        got = got.detach().float().cpu()
        rel = ((got - want).abs().max() / want.abs().max()).item()
        cos = torch.nn.functional.cosine_similarity(got.reshape(1, -1).double(), want.reshape(1, -1).double()).item()
        assert rel < tol and cos > min_cos, (what, rel, cos)
    # element-wise bound = kernel-vs-oracle (<= 6e-2, fp16 deltas) + oracle-vs-golden (<= 2e-2) with margin; the direction
    # of every gradient (cosine) is the sharp criterion
    check(m.field.mlp_base.params.grad, g["mlp_base_grad"], "mlp_base", 0.12)
    check(m.field.mlp_head.params.grad, g["mlp_head_grad"], "mlp_head", 0.12)
    check(m.time_embedding.weight.grad, g["time_emb_grad"], "time_emb", 0.12)
    # deformation branch: the golden is fp32 ('none' precision) while the kernels keep warp codes, activations and
    # deltas in fp16; for the smallest of these gradients (warp codes, |g| ~ 2e-5): rel 0.09, cos 0.993
    check(m.time_embedding_deformation.weight.grad, g["time_emb_deform_grad"], "time_emb_deform", 0.3, 0.97)
    se3 = m.deformation_field.se3_field
    for i, layer in enumerate(se3.mlp_stem.layers):
        check(layer.weight.grad, g[f"stem_w{i}_grad"], f"stem_w{i}", 0.3, 0.97)
        check(layer.bias.grad, g[f"stem_b{i}_grad"], f"stem_b{i}", 0.3, 0.97)
    check(se3.mlp_r.layers[0].weight.grad, g["r_w_grad"], "r_w", 0.3, 0.97)
    check(se3.mlp_v.layers[0].weight.grad, g["v_w_grad"], "v_w", 0.3, 0.97)
    flat = m.field.hash_ensemble.tables.grad.reshape(-1).cpu()
    pick = torch.randint(0, flat.numel(), (200_000,), generator=torch.Generator().manual_seed(5))
    cos = torch.nn.functional.cosine_similarity(flat[pick].reshape(1, -1).double(), g["tables_grad_sample"].reshape(1, -1).double()).item()
    assert cos > 0.99, cos
    assert abs((flat.double() ** 2).sum().item() / g["tables_grad_sums"][1].item() - 1.0) < 0.25


def test_occupancy_update_vs_nerfacc_oracle(monkeypatch):
    """OccGridEstimator._update (a14) against oracle/tp/nerfacc_cpu.OccGridEstimator._update on the SAME random draws
    (torch.rand_like / torch.randint are patched to draw on the CPU from one seeded generator and move to the caller's
    device): two warm-up steps over all cells, then two post-warm-up steps (uniform + occupied cells, WITH duplicate
    cell ids).  Cells evaluated once must agree with the oracle; a cell evaluated k times must hold
    max(old * decay, max of its k candidates) -- a valid outcome of nerfacc's order-dependent indexed assignment."""
    from nersemble_b200.plugin.sampler import OccGridEstimator
    from oracle.tp import nerfacc_cpu
    aabb = torch.tensor([-2.5, -1.8, -2.5, 2.2, 1.8, 2.0])
    res, decay, occ_thre = 64, 0.95, 1e-2
    real_randint = torch.randint

    def occ_fn(x):      # analytic density blob * step: the same float32 arithmetic on both devices up to exp() ulps
        c = torch.tensor([0.1, -0.2, 0.3], device=x.device)
        return 40.0 * torch.exp(-((x - c) ** 2).sum(-1, keepdim=True) / 0.8) * 0.011

    def patch(seed):
        gen = torch.Generator().manual_seed(seed)
        monkeypatch.setattr(torch, "rand_like", lambda t, **kw: torch.rand(t.shape, generator=gen).to(t.device))
        monkeypatch.setattr(torch, "randint", lambda high, size, **kw: real_randint(high, size, generator=gen).to(kw.get("device", "cpu")))

    got = OccGridEstimator(aabb, resolution=res, levels=1).to(DEV).train()
    want = nerfacc_cpu.OccGridEstimator(aabb, resolution=res, levels=1).train()
    n_dup_total = 0
    for step, seed in ((0, 1), (16, 2), (4096, 3), (4112, 4)):
        prev, prev_bin = want.occs.clone(), want.binaries.clone()
        for est in (got, want):
            patch(seed)
            est._update(step=step, occ_eval_fn=occ_fn, occ_thre=occ_thre, ema_decay=decay, warmup_steps=256)
            monkeypatch.undo()
        g_occs = got.occs.cpu()
        if step < 256:
            torch.testing.assert_close(g_occs, want.occs, rtol=2e-6, atol=1e-9)
        else:
            gen = torch.Generator().manual_seed(seed)           # rebuild the draws of _sample_uniform_and_occupied_cells
            n = want.cells_per_lvl // 4
            idx = real_randint(want.cells_per_lvl, (n,), generator=gen)
            occ_idx = torch.nonzero(prev_bin.flatten())[:, 0]
            if n < len(occ_idx):
                occ_idx = occ_idx[real_randint(len(occ_idx), (n,), generator=gen)]
            idx = torch.cat([idx, occ_idx])
            x = (want.grid_coords[idx] + torch.rand((idx.numel(), 3), generator=gen)) / want.resolution
            x = want.aabbs[0, :3] + x * (want.aabbs[0, 3:] - want.aabbs[0, :3])
            amax = (prev * decay).scatter_reduce(0, idx, occ_fn(x).squeeze(-1), reduce="amax", include_self=True)
            cnt = torch.bincount(idx, minlength=want.cells_per_lvl)
            once, touched = cnt == 1, cnt > 0
            n_dup_total += int((cnt > 1).sum())
            torch.testing.assert_close(g_occs[once], want.occs[once], rtol=2e-6, atol=1e-9)      # vs the nerfacc restatement
            torch.testing.assert_close(g_occs[touched], amax[touched], rtol=2e-6, atol=1e-9)    # duplicates: largest candidate
            assert torch.equal(g_occs[~touched], prev[~touched])
            want.occs.copy_(torch.where(touched, amax, prev))
        # threshold / binaries: identical wherever occs is not within rounding of the threshold
        thre = torch.clamp(want.occs[want.occs >= 0].mean(), max=occ_thre)
        want_bin = want.occs > thre
        safe = (want.occs - thre).abs() > 1e-6
        assert torch.equal(got.binaries.cpu().flatten()[safe], want_bin[safe])
        # continue from the CUDA state so that both sides draw the same occupied cells in the next step
        want.occs.copy_(g_occs); want.binaries = got.binaries.cpu().clone()
    assert n_dup_total > 100
    assert 0.0 < float(got.binaries.float().mean()) < 1.0
