"""Generate tests/golden/*.npz by running the REAL reference glue on CPU.

TEST INFRASTRUCTURE.  Only runnable in the build container (needs /root/reference).
    python -m oracle.gen_golden

The reference modules (src/nersemble/nerfstudio/**: NeRSembleNGPModel, NeRSembleNeRFactoField,
HashEnsemble, SE3DeformationField, NeRSembleVolumetricSampler, DeformationRenderer, losses in
models/base.py) are imported unmodified from /root/reference/src; their un-vendored third-party
imports (tinycudann, nerfacc, nerfstudio, torch_efficient_distloss) resolve to the CPU
restatements in oracle/tp.  So the goldens pin the reference's OWN code (rearrange/window/
blend, skip-MLP wiring, SE(3) map, offset quirk, selector, padding, compositing order, losses);
the third-party arithmetic underneath stays [3P-mem] / parity unpinned.

Parameters are NOT stored: each case records the seed/knobs of oracle.pipeline.random_params,
which regenerates them bit-identically; they are copied into the reference model here
(tables converted native -> 8 tcnn grids).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

REF_SRC = "/root/reference/src"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def build_reference_model(P, n_timesteps, log2T, use_frustum=False):
    from nersemble.nerfstudio.models.nersemble_instant_ngp import NeRSembleNGPModel, NeRSembleNGPModelConfig
    from nersemble.nerfstudio.field_components.hash_ensemble import HashEnsembleConfig, TCNNHashEncodingConfig
    from nersemble.nerfstudio.field_components.deformation_field import SE3DeformationFieldConfig
    from nerfstudio.data.scene_box import SceneBox
    from oracle.pipeline import tables_to_tcnn

    # hparams = scripts/train/train_nersemble.py:184-240 (scale_factor 9 -> factor 1)
    cfg = NeRSembleNGPModelConfig(
        render_step_size=0.011, near_plane=0.2, far_plane=1e3, cone_angle=0.0, alpha_thre=1e-2, occ_thre=1e-2,
        early_stop_eps=0, background_color="white", grid_levels=1, disable_scene_contraction=True,
        n_timesteps=n_timesteps, latent_dim_time=32, use_masked_rgb_loss=True, alpha_mask_threshold=0,
        lambda_alpha_loss=1e-2, lambda_near_loss=1e-4, lambda_empty_loss=1e-2, lambda_depth_loss=1e-4,
        lambda_dist_loss=1e-4,
        use_hash_ensemble=True,
        hash_ensemble_config=HashEnsembleConfig(
            n_hash_encodings=32, hash_encoding_config=TCNNHashEncodingConfig(log2_hashmap_size=log2T),
            disable_initial_hash_ensemble=True, use_soft_transition=True),
        use_deformation_field=True, use_separate_deformation_time_embedding=True,
        deformation_field_config=SE3DeformationFieldConfig(warp_code_dim=128, mlp_num_layers=6, mlp_layer_width=128),
        window_hash_encodings_begin=40000, window_hash_encodings_end=80000,
        window_deform_begin=0, window_deform_end=20000, use_view_frustum_culling=False)
    model = NeRSembleNGPModel(cfg, scene_box=SceneBox(P.aabb.clone()), num_train_data=16,
                              metadata={"camera_frustums": None})
    with torch.no_grad():
        for c, g in enumerate(tables_to_tcnn(P.tables)):
            model.field.hash_ensemble.hash_encodings[c].params.copy_(g)
        model.field.mlp_base.params.copy_(torch.cat([w.reshape(-1) for w in P.base_w]))
        model.field.mlp_head.params.copy_(torch.cat([w.reshape(-1) for w in P.head_w]))
        se3 = model.deformation_field.se3_field
        for i, layer in enumerate(se3.mlp_stem.layers):
            layer.weight.copy_(P.deform_w[i]); layer.bias.copy_(P.deform_b[i])
        se3.mlp_r.layers[0].weight.copy_(P.r_w); se3.mlp_r.layers[0].bias.copy_(P.r_b)
        se3.mlp_v.layers[0].weight.copy_(P.v_w); se3.mlp_v.layers[0].bias.copy_(P.v_b)
        model.time_embedding.weight.copy_(P.time_emb)
        model.time_embedding_deformation.weight.copy_(P.time_emb_deform)
    return model


def ring_rays(R, seed, n_cams=16, radius=9.0, spread=1.2):
    """Synthetic pinhole rays from cameras on a ring of radius 9 aimed near the origin
    (SURVEY 8d config 2; scale_factor 9, train_nersemble.py:124)."""
    g = torch.Generator().manual_seed(seed)
    cam = torch.randint(0, n_cams, (R,), generator=g)
    ang = cam.float() / n_cams * 2 * torch.pi
    o = torch.stack([radius * torch.sin(ang), 0.3 * torch.cos(3 * ang), radius * torch.cos(ang)], -1)
    target = (torch.rand((R, 3), generator=g) * 2 - 1) * spread
    d = target - o
    d = d / d.norm(dim=-1, keepdim=True)
    times = torch.rand((R, 1), generator=g)
    return o.float(), d.float(), times.float(), cam.long()[:, None]


def blob_grid(seed, res=128, n_blobs=6):
    g = torch.Generator().manual_seed(seed)
    c = torch.rand((n_blobs, 3), generator=g) * 0.6 + 0.2
    rad = torch.rand((n_blobs,), generator=g) * 0.15 + 0.08
    ax = (torch.arange(res).float() + 0.5) / res
    X, Y, Z = torch.meshgrid(ax, ax, ax, indexing="ij")
    pts = torch.stack([X, Y, Z], -1)
    occ = torch.zeros(res, res, res, dtype=torch.bool)
    for i in range(n_blobs):
        occ |= ((pts - c[i]) ** 2).sum(-1) < rad[i] ** 2
    return occ


class FixedSampler(torch.nn.Module):
    """Stands in for model.sampler to impose BASELINE config-1 fixed samples (no occ-grid)."""

    def __init__(self, t_starts, t_ends, ray_indices):
        super().__init__()
        self.ts, self.te, self.ri = t_starts, t_ends, ray_indices

    def forward(self, ray_bundle, **kw):
        from nerfstudio.cameras.rays import Frustums, RaySamples
        ri = self.ri
        o = ray_bundle.origins[ri]; d = ray_bundle.directions[ri]
        rs = RaySamples(frustums=Frustums(origins=o, directions=d, starts=self.ts[:, None], ends=self.te[:, None],
                                          pixel_area=torch.zeros_like(o[:, :1])),
                        camera_indices=ray_bundle.camera_indices[ri])
        rs.times = ray_bundle.times[ri]
        return rs, ri


def run_case(name, *, mode, R, T, log2T, table_scale, time_std_scale, deform_last_scale, w_hash, w_deform,
             sampler, training=False, n_fixed=64, rays_seed=1, grid_seed=None, autocast=False):
    from oracle.tp.tcnn_cpu import Precision
    from oracle import pipeline as pl
    from nerfstudio.cameras.rays import RayBundle
    Precision.mode = mode
    Precision.autocast = autocast
    knobs = dict(seed=19980801, n_timesteps=T, log2_hashmap_size=log2T, table_scale=table_scale,
                 time_std_scale=time_std_scale, deform_last_scale=deform_last_scale)
    P = pl.random_params(**knobs)
    model = build_reference_model(P, T, log2T)
    model.sched_window_hash_encodings.value = w_hash
    model.sched_window_deform.value = w_deform
    o, d, times, cams = ring_rays(R, rays_seed)
    if T == 1:
        times = torch.zeros_like(times)
    rb = RayBundle(origins=o, directions=d, pixel_area=torch.ones(R, 1), camera_indices=cams, times=times)
    extra = {}
    if sampler == "fixed":
        ts, te, ri = pl.fixed_samples(o, d, P.aabb, n_fixed, 0.011, near=0.2)
        model.sampler = FixedSampler(ts, te, ri)
    else:
        occ = blob_grid(grid_seed)
        model.occupancy_grid.binaries[0] = occ
        # a plausible EMA state so that occs.mean() (visibility threshold) is defined
        model.occupancy_grid.occs.copy_(occ.flatten().float() * 0.05)
        extra["grid_seed"] = grid_seed
    model.train(training)
    if training:
        torch.manual_seed(4242)   # jitter = torch.rand(R) * step drawn first inside sampling()
        extra["jitter_seed"] = 4242
    with torch.no_grad():
        out = model.get_outputs(rb)
    rs = out["ray_samples"][0]
    res = {
        "origins": o, "directions": d, "times": times, "camera_indices": cams,
        "rgb": out["rgb"], "accumulation": out["accumulation"], "depth": out["depth"],
        "deformation": out["deformation"], "num_samples_per_ray": out["num_samples_per_ray"],
        "weights": out["weights"][0], "ray_indices": out["ray_indices"][0],
        "t_starts": rs.frustums.starts[:, 0], "t_ends": rs.frustums.ends[:, 0], "offsets": rs.frustums.offsets,
    }
    meta = dict(name=name, mode=mode, autocast=autocast, R=R, knobs=knobs, w_hash=w_hash, w_deform=w_deform,
                sampler=sampler, training=training, n_fixed=n_fixed, rays_seed=rays_seed, **extra)
    save(name, res, meta)
    return model, P, rb, out


def save(name, tensors, meta):
    os.makedirs(OUT, exist_ok=True)
    arrs = {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in tensors.items()}
    arrs["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **arrs)
    print("wrote", name, {k: v.shape for k, v in arrs.items() if k != "meta_json"})


def density_case(name, mode):
    from oracle.tp.tcnn_cpu import Precision
    from oracle import pipeline as pl
    Precision.mode = mode; Precision.autocast = False
    T, log2T = 4, 14
    knobs = dict(seed=19980801, n_timesteps=T, log2_hashmap_size=log2T, table_scale=0.5,
                 time_std_scale=100.0, deform_last_scale=1e-3)
    P = pl.random_params(**knobs)
    model = build_reference_model(P, T, log2T)
    model.sched_window_hash_encodings.value = 20.25
    model.sched_window_deform.value = 5.5
    g = torch.Generator().manual_seed(7)
    lo, hi = P.aabb[0], P.aabb[1]
    pos = lo + (torch.rand((256, 3), generator=g) * 1.2 - 0.1) * (hi - lo)    # some points outside the box
    times = torch.randint(0, T, (256, 1), generator=g).float() / (T - 1)
    with torch.no_grad():
        sigma = model.field_density_fn(pos, times)
    save(name, {"positions": pos, "times": times, "density": sigma},
         dict(name=name, mode=mode, knobs=knobs, w_hash=20.25, w_deform=5.5))


def loss_case(name):
    """get_loss_dict (models/nersemble_instant_ngp.py:366-407 -> models/base.py:90-249) in training mode."""
    trained = dict(table_scale=0.5, time_std_scale=100.0, deform_last_scale=1e-3)
    model, P, rb, out = run_case(name + "_render", mode="none", R=40, T=4, log2T=14, w_hash=32.0, w_deform=7.0,
                                 sampler="occ", grid_seed=5, training=True, **trained)
    R = 40
    g = torch.Generator().manual_seed(11)
    batch = {
        "image": torch.rand((R, 3), generator=g),
        "alpha_map": torch.randint(0, 256, (R, 1), generator=g).float(),
        "depth_maps": torch.where(torch.rand((R,), generator=g) < 0.8,
                                  7.5 + 2.0 * torch.rand((R,), generator=g), torch.zeros(R)),
    }
    batch["alpha_map"][:5] = 255.0
    model.sched_eps_depth.value = 0.35
    ld = model.get_loss_dict(out, batch)
    tensors = {("loss_" + k): v for k, v in ld.items()}
    tensors.update({("batch_" + k): v for k, v in batch.items()})
    save(name, tensors, dict(name=name, eps_depth=0.35, render_case=name + "_render"))


def grad_case(name):
    """Parameter GRADIENTS of one full training step computed by torch autograd through the unmodified reference glue
    (NeRSembleNGPModel.get_outputs -> get_loss_dict -> backward) on the CPU stand-ins: pins the backward kernels and
    the oracle's own autograd.  Samples are deterministic (sampler.eval(): no jitter, no pre-pass); all six losses."""
    from oracle.tp.tcnn_cpu import Precision
    from oracle import pipeline as pl
    from nerfstudio.cameras.rays import RayBundle
    Precision.mode = "none"; Precision.autocast = False
    knobs = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0, deform_last_scale=0.02)
    P = pl.random_params(**knobs)
    model = build_reference_model(P, 4, 14)
    w_hash, w_deform, R = 32.0, 5.5, 48
    model.sched_window_hash_encodings.value = w_hash
    model.sched_window_deform.value = w_deform
    o, d, times, cams = ring_rays(R, 21)
    rb = RayBundle(origins=o, directions=d, pixel_area=torch.ones(R, 1), camera_indices=cams, times=times)
    occ = blob_grid(3)
    model.occupancy_grid.binaries[0] = occ
    model.occupancy_grid.occs.copy_(occ.flatten().float() * 0.05)
    model.train(True)
    model.sampler.eval()
    g = torch.Generator().manual_seed(11)
    batch = {"image": torch.rand((R, 3), generator=g), "alpha_map": torch.randint(0, 256, (R, 1), generator=g).float(),
             "depth_maps": torch.where(torch.rand((R,), generator=g) < 0.8, 7.5 + 2.0 * torch.rand((R,), generator=g), torch.zeros(R))}
    batch["alpha_map"][:5] = 255.0
    model.sched_eps_depth.value = 0.35
    out = model.get_outputs(rb)
    ld = model.get_loss_dict(out, batch)
    sum(ld.values()).backward()
    from oracle.pipeline import tables_from_tcnn
    gt = tables_from_tcnn([m.params.grad for m in model.field.hash_ensemble.hash_encodings])     # [entries, 32, 2]
    # the dense table gradient is 63 MB (8 M non-zeros): the fixture keeps a seeded random sample of 200 k elements
    # (zeros included), the global sums, and the squared norm per level
    flat = gt.reshape(-1)
    pick = torch.randint(0, flat.numel(), (200_000,), generator=torch.Generator().manual_seed(5))
    from oracle.tp.tcnn_cpu import hashgrid_levels
    lv = hashgrid_levels(16, 14, 16, 1.4472692012786865)
    offs = [int(v) for v in lv.offset]          # [L + 1], entry units
    per_level = torch.stack([(gt[offs[l]:offs[l + 1]].double() ** 2).sum() for l in range(16)])
    se3 = model.deformation_field.se3_field
    tensors = {"origins": o, "directions": d, "times": times, "camera_indices": cams,
               "ray_indices": out["ray_indices"][0], "tables_grad_sample": flat[pick],
               "tables_grad_sums": torch.stack([flat.double().sum(), (flat.double() ** 2).sum(), flat.double().abs().sum()]),
               "tables_grad_sq_per_level": per_level, "tables_grad_nonzeros": torch.tensor(int((flat != 0).sum())),
               "mlp_base_grad": model.field.mlp_base.params.grad, "mlp_head_grad": model.field.mlp_head.params.grad,
               "time_emb_grad": model.time_embedding.weight.grad, "time_emb_deform_grad": model.time_embedding_deformation.weight.grad,
               "r_w_grad": se3.mlp_r.layers[0].weight.grad, "r_b_grad": se3.mlp_r.layers[0].bias.grad,
               "v_w_grad": se3.mlp_v.layers[0].weight.grad, "v_b_grad": se3.mlp_v.layers[0].bias.grad}
    for i, layer in enumerate(se3.mlp_stem.layers):
        tensors[f"stem_w{i}_grad"] = layer.weight.grad
        tensors[f"stem_b{i}_grad"] = layer.bias.grad
    tensors.update({("loss_" + k): v.detach() for k, v in ld.items()})
    tensors.update({("batch_" + k): v for k, v in batch.items()})
    save(name, tensors, dict(name=name, knobs=knobs, R=R, w_hash=w_hash, w_deform=w_deform, grid_seed=3, rays_seed=21,
                             eps_depth=0.35, table_entries=int(gt.shape[0])))


def main():
    sys.path.insert(0, REF_SRC)
    sys.path.insert(0, os.path.dirname(HERE))
    from oracle.tp import install_stubs
    install_stubs()
    if len(sys.argv) > 1 and sys.argv[1] == "grads":     # only the gradient golden (the others are unchanged)
        grad_case("grads_train")
        return
    init = dict(table_scale=1e-4, time_std_scale=1.0, deform_last_scale=1e-5)
    trained = dict(table_scale=0.5, time_std_scale=100.0, deform_last_scale=1e-3)
    # BASELINE config 1: 32 rays x 64 samples, 1 timestep, no occ-grid, full-size tables
    run_case("config1_init_reference", mode="reference", R=32, T=1, log2T=19, w_hash=32.0, w_deform=7.0,
             sampler="fixed", **init)
    run_case("config1_trained_none", mode="none", R=32, T=1, log2T=19, w_hash=32.0, w_deform=7.0,
             sampler="fixed", **trained)
    for mode in ("reference", "kernel", "none"):
        run_case(f"fixed_trained_{mode}", mode=mode, R=32, T=4, log2T=14, w_hash=32.0, w_deform=7.0,
                 sampler="fixed", **trained)
    run_case("fixed_trained_autocast", mode="reference", autocast=True, R=32, T=4, log2T=14, w_hash=32.0,
             w_deform=7.0, sampler="fixed", **trained)
    run_case("occ_eval_soft", mode="none", R=48, T=4, log2T=14, w_hash=1.5, w_deform=3.3,
             sampler="occ", grid_seed=3, **trained)
    run_case("occ_eval_whash1", mode="none", R=48, T=4, log2T=14, w_hash=1, w_deform=0.0,
             sampler="occ", grid_seed=4, **trained)
    run_case("occ_train_prepass", mode="none", R=48, T=4, log2T=14, w_hash=32.0, w_deform=7.0,
             sampler="occ", grid_seed=5, training=True, **trained)
    density_case("density_fn_none", "none")
    density_case("density_fn_kernel", "kernel")
    loss_case("losses_train")
    grad_case("grads_train")


if __name__ == "__main__":
    main()
