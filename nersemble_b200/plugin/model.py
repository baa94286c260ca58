"""NeRSembleNGPModel -- mirror of models/nersemble_instant_ngp.py:39-516 and models/base.py:15-249."""
from __future__ import annotations

from dataclasses import dataclass, field
from math import sqrt
from typing import Dict, List, Optional, Tuple, Type

import torch
from torch import Tensor, nn
from torch.nn import Parameter, init

from .. import ops
from ..nerfstudio_shim import (FieldHeadNames, Model, RayBundle, RaySamples, SceneBox, TrainingCallback,
                               TrainingCallbackAttributes, TrainingCallbackLocation)
from .components import GenericScheduler, HashEnsembleConfig, SE3DeformationField, SE3DeformationFieldConfig
from .field import NeRSembleNeRFactoField
from .sampler import NeRSembleVolumetricSampler, OccGridEstimator


@dataclass
class BaseModelConfig:
    """models/base.py:15-32 (+ the nerfstudio ModelConfig fields the scripts touch)."""
    enable_collider: bool = False
    collider_params: Optional[Dict[str, float]] = None
    loss_coefficients: Optional[Dict[str, float]] = None
    eval_num_rays_per_chunk: int = 4096
    use_masked_rgb_loss: bool = False
    alpha_mask_threshold: float = 0.5
    lambda_alpha_loss: float = 0
    lambda_empty_loss: float = 0
    lambda_near_loss: float = 0
    lambda_depth_loss: float = 0
    eps_depth_initial: float = 0.9
    eps_depth_final: float = 0.01
    eps_depth_begin_step: int = 0
    eps_depth_end_step: int = 10000
    lambda_dist_loss: float = 0
    dist_loss_max_rays: int = 5000


@dataclass
class NeRSembleNGPModelConfig(BaseModelConfig):
    """models/nersemble_instant_ngp.py:39-75 on top of nerfstudio InstantNGPModelConfig's defaults."""
    _target: Type = field(default_factory=lambda: NeRSembleNGPModel)
    # InstantNGPModelConfig
    grid_resolution: int = 128
    grid_levels: int = 4
    max_res: int = 2048
    log2_hashmap_size: int = 19
    alpha_thre: float = 0.01
    cone_angle: float = 0.004
    render_step_size: Optional[float] = None
    near_plane: float = 0.05
    far_plane: float = 1e3
    use_appearance_embedding: bool = False
    background_color: str = "random"
    disable_scene_contraction: bool = False
    # NeRSemble
    n_timesteps: int = 1
    latent_dim_time: int = 128
    spherical_harmonics_degree: int = 0
    use_hash_ensemble: bool = False
    hash_ensemble_config: Optional[HashEnsembleConfig] = None
    use_deformation_field: bool = False
    deformation_field_config: Optional[SE3DeformationFieldConfig] = None
    use_separate_deformation_time_embedding: bool = True
    window_deform_begin: int = 0
    window_deform_end: int = 0
    window_hash_encodings_begin: int = 0
    window_hash_encodings_end: int = 1
    early_stop_eps: float = 1e-4
    occ_thre: float = 1e-2
    disable_occupancy_grid: bool = False
    occupancy_grid_ema_decay: float = 0.95
    occupancy_grid_warmup_steps: int = 256
    max_n_samples_per_batch: int = -1
    use_view_frustum_culling: bool = False
    view_frustum_culling: int = 2

    def setup(self, **kwargs):
        return self._target(self, **kwargs)


class _RenderFunction(torch.autograd.Function):
    """Differentiable fused render (training).  Forward = nsb_field_forward (saving the blended features, the warped
    positions and the deformation activations) + nsb_composite_forward; backward = nsb_composite_backward ->
    nsb_field_backward -> nsb_deform_backward, with the fp32 gradients mapped back to the reference's parameter
    layouts (flat tcnn MLP params, nn.Linear weights/biases, the two time embeddings; the hash tables in native layout)."""

    @staticmethod
    def forward(ctx, model, origins, directions, ray_times, starts, ends, ray_indices, packed_info, wh, wd, *params):
        P = model.native_params()
        deform = model.config.use_deformation_field
        kw = dict(origins=origins, directions=directions, ray_times=ray_times, t_starts=starts, t_ends=ends,
                  ray_indices=ray_indices)
        reuse = getattr(model, "_prepass_payload", None)       # (feat, corner_vals) of exactly these samples, or None
        model._prepass_payload = None
        if reuse is not None and reuse[0].shape[0] == starts.shape[0]:
            want = ("sigma", "rgb", "xs") + (("offsets", "deform_acts") if deform else ())
            f = ops.field_forward(P, window_hash=wh, window_deform=wd, use_deformation=deform, want=want, given_feat=reuse[0],
                                  **kw, **model._blend_opts())
            f["feat"], f["corner_vals"] = reuse
        else:
            want = ("sigma", "rgb", "feat", "xs") + (("offsets", "deform_acts", "corner_vals") if deform else ())
            f = ops.field_forward(P, window_hash=wh, window_deform=wd, use_deformation=deform, want=want, **kw,
                                  **model._blend_opts())
        c = ops.composite(packed_info, starts, ends, f["sigma"], f["rgb"], f["offsets"] if deform else None, training=True)
        ctx.model, ctx.P, ctx.kw, ctx.wh, ctx.wd, ctx.deform = model, P, kw, wh, wd, deform
        ctx.saved = {k: f[k] for k in ("feat", "xs", "sigma", "rgb")}
        if deform:
            ctx.saved.update(deform_acts=f["deform_acts"], deform_enc=f["deform_enc"], corner_vals=f["corner_vals"])
        elif "corner_vals" in f:
            ctx.saved.update(corner_vals=f["corner_vals"])
        ctx.packed_info, ctx.workspace = packed_info, c["workspace"]
        outs = (c["rgb"], c["accumulation"], c["depth"], c["weights"])
        if deform:
            ctx.mark_non_differentiable(f["offsets"], c["deformation"])
            outs += (c["deformation"], f["offsets"])
        return outs

    @staticmethod
    def backward(ctx, g_rgb, g_acc, g_depth, g_weights, *unused):
        from .. import packing
        model, kw = ctx.model, ctx.kw
        if g_rgb is None:                       # a loss that does not touch rgb (e.g. only the distortion term)
            g_rgb = torch.zeros((ctx.packed_info.shape[0], 3), dtype=torch.float32, device=ctx.saved["sigma"].device)
        ls = float(getattr(model, "mlp_loss_scale", 128.0))
        d_sigma, d_rgb = ops.composite_backward(ctx.packed_info, kw["t_starts"], kw["t_ends"], ctx.saved["sigma"],
                                                ctx.saved["rgb"], ctx.workspace, g_rgb,
                                                None if g_acc is None else g_acc.reshape(-1),
                                                None if g_depth is None else g_depth.reshape(-1),
                                                None if g_weights is None else g_weights.reshape(-1))
        he = model.field.hash_ensemble
        defer = he.defer_table_grad and he.pending_table_grad is None     # a second backward before step() goes dense
        g = ops.field_backward(ctx.P, ctx.saved, d_sigma, d_rgb, window_hash=ctx.wh, loss_scale=ls, want_dx=ctx.deform,
                               defer_tables=defer, **kw, **model._blend_opts())
        if "pending" in g:
            he.pending_table_grad = g["pending"]
            # GradScaler contract (SURVEY 8b): the parked table gradient is no `.grad`, so the scaler's inf check cannot
            # see it.  Its entries are sums of |w| <= 1 times d_feat, so d_feat is finite iff it is: fold that flag into
            # a gradient the scaler DOES check (x - x = 0 for finite x, NaN otherwise) -- no host synchronisation.
            flag = g["d_feat"].sum()
            g["d_base_w"] = g["d_base_w"] + (flag - flag)
            hook = getattr(he, "table_grad_hook", None)
            if hook is not None:          # distributed.overlap_table_allreduce: the collective overlaps the rest of the backward
                hook(he)
        grads = [g.get("d_tables"), g["d_base_w"], g["d_head_w"], g["d_blend_codes"]]
        if ctx.deform:
            d = ops.deform_backward(ctx.P, ctx.saved, g["d_xs"], window_deform=ctx.wd, loss_scale=ls, **kw)
            grads.append(d["d_warp_codes"])
            for l in range(6):
                grads += [d["d_stem_w"][l], d["d_stem_b"][l]]
            grads += [d["d_r_w"], d["d_r_b"], d["d_v_w"], d["d_v_b"]]
        return (None,) * 10 + tuple(grads)


class _FusedLosses(torch.autograd.Function):
    """nsb_losses_forward / nsb_losses_backward behind autograd: values [6] in ops.LOSS_NAMES order."""

    @staticmethod
    def forward(ctx, rgb, acc, depth, weights, packed_info, starts, ends, image, alpha, depth_target, cfg):
        values, state = ops.losses_forward(packed_info, starts, ends, weights, rgb, acc, depth, image, alpha, depth_target, cfg)
        ctx.state = state
        ctx.shapes = (rgb.shape, acc.shape, depth.shape, weights.shape)
        return values

    @staticmethod
    def backward(ctx, g_values):
        d_rgb, d_acc, d_depth, d_w = ops.losses_backward(ctx.state, g_values)
        s = ctx.shapes
        return (d_rgb.reshape(s[0]), d_acc.reshape(s[1]), d_depth.reshape(s[2]), d_w.reshape(s[3])) + (None,) * 7


def _segment_exclusive_sum(x: Tensor, ray_indices: Tensor, n_rays: int) -> Tensor:
    cnt = torch.zeros(n_rays, dtype=torch.long, device=x.device).index_add_(0, ray_indices, torch.ones_like(ray_indices))
    starts = cnt.cumsum(0) - cnt
    inc = torch.cumsum(x.double(), 0)
    before = torch.cat([torch.zeros(1, dtype=torch.float64, device=x.device), inc])[starts]
    return (inc - x.double() - before[ray_indices]).to(x.dtype)


class NeRSembleNGPModel(Model):
    """Subclass of nerfstudio's `Model` (the real class when nerfstudio is importable, the 0.3.1-shaped stand-in of
    nerfstudio_shim otherwise): the base constructor stores config / scene_box / num_train_data / kwargs, calls
    populate_modules() and creates device_indicator_param, exactly as under VanillaPipeline (train_nersemble.py:163,184)."""
    config: NeRSembleNGPModelConfig

    def __init__(self, config: NeRSembleNGPModelConfig, scene_box: SceneBox, num_train_data: int, **kwargs):
        super().__init__(config=config, scene_box=scene_box, num_train_data=num_train_data, **kwargs)
        self._native = None
        self._native_version = None
        self.sync_free_losses = True     # get_loss_dict without host syncs on CUDA (see _loss_dict_sync_free)
        self.fused_losses = True         # ... and, when the outputs come from get_outputs, in fused kernels (_loss_dict_fused)
        self.lpips = None                # optional callable(image[1,3,H,W], rgb[1,3,H,W]) -> scalar (needs pretrained weights)
        self.use_fused_render = True     # eval renders: sampler -> field -> composite fused, no host sync (ops.render_rays)
        self.use_fused_sampler = True    # training: march / density pre-pass / visibility / packing with one host sync
        self.frame_tables = True         # eval renders gather member-blended tables: per frame (one timestep per camera
                                         # frame) or per timestep (mixed-time bundles); False: per-sample blend of the lines
        self.frame_table_min_rays = 16384  # ... for frames of at least this many rays (the check is one host sync per frame,
                                           # the table one streaming pass over the hash tables)
        self.prepass_reuse = True        # ... and the pre-pass's blended features / corner values are packed with the kept
                                         # samples, so the differentiable forward does not gather the tables a second time

    def populate_modules(self):
        """models/nersemble_instant_ngp.py:81-179 (+ BaseModel.populate_modules, base.py:38-47)."""
        cfg = self.config
        if cfg.use_hash_ensemble:
            # hash_ensemble.py:115-117 asserts this at forward time; here the embedding rows ARE the kernel's blend codes
            assert cfg.latent_dim_time == cfg.hash_ensemble_config.n_hash_encodings, \
                "If blend mixing type is chosen, conditioning code needs to have as many dimensions as there are " \
                f"hashtables in the encoding (latent_dim_time={cfg.latent_dim_time}, " \
                f"n_hash_encodings={cfg.hash_ensemble_config.n_hash_encodings})"
        if cfg.lambda_empty_loss > 0 or cfg.lambda_near_loss > 0:
            self.sched_eps_depth = GenericScheduler(cfg.eps_depth_initial, cfg.eps_depth_final, cfg.eps_depth_begin_step,
                                                    cfg.eps_depth_end_step)
        else:
            self.sched_eps_depth = None
        if not cfg.disable_scene_contraction:
            raise NotImplementedError("scene contraction (the NeRSemble recipe sets disable_scene_contraction=True)")
        if cfg.background_color != "white":
            raise NotImplementedError("only background_color='white' (train_nersemble.py:193)")
        self.field = NeRSembleNeRFactoField(
            aabb=self.scene_box.aabb, num_images=self.num_train_data, log2_hashmap_size=cfg.log2_hashmap_size,
            max_res=cfg.max_res, spatial_distortion=None, spherical_harmonics_degree=cfg.spherical_harmonics_degree,
            use_hash_ensemble=cfg.use_hash_ensemble, hash_ensemble_config=cfg.hash_ensemble_config,
            use_appearance_embedding=cfg.use_appearance_embedding, max_n_samples_per_batch=cfg.max_n_samples_per_batch)
        self.deformation_field = None
        if cfg.use_deformation_field:
            self.deformation_field = SE3DeformationField(self.scene_box.aabb, cfg.deformation_field_config,
                                                         max_n_samples_per_batch=cfg.max_n_samples_per_batch)
        self.time_embedding = None
        if cfg.use_deformation_field or cfg.use_hash_ensemble:
            self.time_embedding = nn.Embedding(cfg.n_timesteps, cfg.latent_dim_time)
            init.normal_(self.time_embedding.weight, mean=0., std=0.01 / sqrt(cfg.latent_dim_time))
            if cfg.use_separate_deformation_time_embedding:
                self.time_embedding_deformation = nn.Embedding(cfg.n_timesteps, cfg.deformation_field_config.warp_code_dim)
                init.normal_(self.time_embedding_deformation.weight, mean=0.,
                             std=0.01 / sqrt(cfg.deformation_field_config.warp_code_dim))
        self.scene_aabb = Parameter(self.scene_box.aabb.flatten(), requires_grad=False)
        if cfg.render_step_size is None:
            cfg.render_step_size = ((self.scene_aabb[3:] - self.scene_aabb[:3]) ** 2).sum().sqrt().item() / 1000
        self.occupancy_grid = OccGridEstimator(roi_aabb=self.scene_aabb, resolution=cfg.grid_resolution, levels=cfg.grid_levels)
        self.sampler = NeRSembleVolumetricSampler(
            occupancy_grid=self.occupancy_grid, density_fn=self.field_density_fn, scene_aabb=self.scene_box.aabb,
            camera_frustums=self.kwargs.get('metadata', {}).get('camera_frustums'),
            view_frustum_culling=cfg.view_frustum_culling if cfg.use_view_frustum_culling else None)
        self.sched_window_deform = None
        if cfg.window_deform_end >= 1:
            self.sched_window_deform = GenericScheduler(0, cfg.deformation_field_config.n_freq_pos,
                                                        cfg.window_deform_begin, cfg.window_deform_end)
        self.sched_window_hash_encodings = None
        if cfg.use_hash_ensemble and cfg.window_hash_encodings_end > 0:
            self.sched_window_hash_encodings = GenericScheduler(1, cfg.hash_ensemble_config.n_hash_encodings,
                                                                cfg.window_hash_encodings_begin, cfg.window_hash_encodings_end)

    # ------------------------------------------------------------------ native parameter cache
    def native_params(self) -> ops.NativeParams:
        params = [p for p in self.parameters()]
        v = tuple((p._version, p.data_ptr()) for p in params)
        if self._native is None or v != self._native_version:
            with torch.no_grad():
                cfg = self.config
                deform = self.deformation_field.se3_field.deform_dict() if self.deformation_field is not None else None
                if cfg.use_separate_deformation_time_embedding and self.deformation_field is not None:
                    ted = self.time_embedding_deformation.weight
                else:
                    ted = self.time_embedding.weight if deform is not None else None
                self._native = ops.NativeParams.build(
                    tables=None, time_emb=self.time_embedding.weight, aabb=self.scene_box.aabb, levels=self.field.hash_ensemble.levels,
                    base_w=self.field.base_weights(), head_w=self.field.head_weights(), deform=deform, time_emb_deform=ted,
                    device=self.scene_aabb.device)
            self._native_version = v
        self._native.tables = self.field.hash_ensemble.native_tables()
        return self._native

    def _windows(self):
        wh = self.sched_window_hash_encodings.value if self.sched_window_hash_encodings is not None else None
        wd = self.sched_window_deform.value if self.sched_window_deform is not None else None
        return wh, wd

    def _blend_opts(self):
        he = self.field.hash_ensemble
        return dict(disable_initial=he.disable_initial_hash_ensemble, soft_transition=he.use_soft_transition)

    # ------------------------------------------------------------------ callbacks
    def get_training_callbacks(self, training_callback_attributes: TrainingCallbackAttributes) -> List[TrainingCallback]:
        """models/nersemble_instant_ngp.py:181-233."""

        def update_occupancy_grid(step: int):
            self.occupancy_grid.update_every_n_steps(
                step=step,
                occ_eval_fn=lambda x: self.field_density_fn(
                    x, torch.randint(0, self.config.n_timesteps, (x.shape[0], 1), dtype=torch.int, device=x.device) / (
                        self.config.n_timesteps - 1)) * self.config.render_step_size,
                n=16, occ_thre=self.config.occ_thre, ema_decay=self.config.occupancy_grid_ema_decay,
                warmup_steps=self.config.occupancy_grid_warmup_steps)

        callbacks = [TrainingCallback(where_to_run=[TrainingCallbackLocation.BEFORE_TRAIN_ITERATION],
                                      update_every_num_iters=1, func=update_occupancy_grid)]

        def update_window_param(sched: GenericScheduler, name: str, step: int):
            sched.update(step)

        for sched, name in ((self.sched_window_deform, "sched_window_deform"),
                            (self.sched_window_hash_encodings, "sched_window_hash_encodings"),
                            (self.sched_eps_depth, "sched_eps_depth")):
            if sched is not None:
                callbacks.append(TrainingCallback(where_to_run=[TrainingCallbackLocation.BEFORE_TRAIN_ITERATION],
                                                  update_every_num_iters=1, func=update_window_param, args=[sched, name]))
        return callbacks

    # ------------------------------------------------------------------ density / outputs
    def field_density_fn(self, positions: Tensor, times: Optional[Tensor]) -> Tensor:
        """models/nersemble_instant_ngp.py:235-266: one fused density-only kernel launch."""
        if self.config.disable_occupancy_grid:
            return torch.ones((positions.shape[0],), dtype=positions.dtype, device=positions.device)
        assert times is not None, "Times need to be provided to NeRSemble's density_fn"
        wh, wd = self._windows()
        out = ops.field_forward(self.native_params(), window_hash=wh, window_deform=wd,
                                use_deformation=self.config.use_deformation_field, positions=positions,
                                sample_times=times.reshape(-1).float(), want=("sigma",), **self._blend_opts())
        return out["sigma"][:, None]

    def _ray_times(self, ray_bundle: RayBundle) -> Tensor:
        if ray_bundle.times is not None:
            return ray_bundle.times.reshape(-1).float()
        return ray_bundle.metadata['timesteps'].reshape(-1).float() / max(self.config.n_timesteps - 1, 1)

    def _fused_render(self, ray_bundle: RayBundle, uniform_time: Optional[float] = None) -> "ops.RenderResult":
        """Eval render of a (flat) ray bundle through nsb_render_forward: the nerfacc occupancy march as one cooperative
        launch + field and compositing fused into one launch; the packed sample count stays on the device.
        uniform_time: every ray of the bundle carries this time (a camera frame) -> per-frame blended table."""
        cfg = self.config
        wh, wd = self._windows()
        near_planes, far_planes = self.sampler.eval_planes(ray_bundle, cfg.near_plane, cfg.far_plane)
        og = self.occupancy_grid
        return ops.render_rays(self.native_params(), ray_bundle.origins.reshape(-1, 3), ray_bundle.directions.reshape(-1, 3),
                               self._ray_times(ray_bundle), window_hash=wh, window_deform=wd,
                               use_deformation=cfg.use_deformation_field, training=self.training, sampler="occupancy",
                               near_planes=near_planes, far_planes=far_planes, binaries=og.binaries, aabbs=og.aabbs,
                               step=cfg.render_step_size, cone_angle=cfg.cone_angle, uniform_time=uniform_time,
                               line_gather=not self.frame_tables, **self._blend_opts())

    @torch.no_grad()
    def _sample_packed(self, ray_bundle: RayBundle, jitter: Optional[Tensor], want_payload: bool = False):
        """The sampler call of get_outputs (models/nersemble_instant_ngp.py:283-291) through
        NeRSembleVolumetricSampler.sample_packed: (RaySamples, ray_indices, packed_info) with one host synchronisation."""
        from ..nerfstudio_shim import Frustums
        cfg = self.config
        wh, wd = self._windows()
        o = ray_bundle.origins.reshape(-1, 3).contiguous()
        d = ray_bundle.directions.reshape(-1, 3).contiguous()
        ray_times = self._ray_times(ray_bundle)

        def sigma_packed(cand):
            """field_density_fn (:235-266) on the candidates' midpoints, sample count read on the device."""
            if cfg.disable_occupancy_grid:
                return torch.ones((cand["capacity"],), dtype=torch.float32, device=o.device), None
            reuse = self.prepass_reuse and want_payload
            f = ops.field_forward(self.native_params(), window_hash=wh, window_deform=wd, use_deformation=cfg.use_deformation_field,
                                  origins=o, directions=d, ray_times=ray_times, t_starts=cand["t_starts"], t_ends=cand["t_ends"],
                                  ray_indices=cand["ray_indices"], n_samples_dev=cand["n_total"],
                                  want=("sigma", "feat", "corner_vals") if reuse else ("sigma",), **self._blend_opts())
            return f["sigma"], ({"feat": f["feat"], "corner_vals": f["corner_vals"]} if reuse else None)

        s = self.sampler.sample_packed(ray_bundle, render_step_size=cfg.render_step_size, near_plane=cfg.near_plane,
                                       far_plane=cfg.far_plane, alpha_thre=cfg.alpha_thre, cone_angle=cfg.cone_angle,
                                       early_stop_eps=cfg.early_stop_eps, jitter=jitter, sigma_packed_fn=sigma_packed)
        ri = s["ray_indices"].long()
        origins = o[ri]
        ci = ray_bundle.camera_indices
        ray_samples = RaySamples(frustums=Frustums(origins=origins, directions=d[ri], starts=s["t_starts"][:, None],
                                                   ends=s["t_ends"][:, None], pixel_area=torch.zeros_like(origins[:, :1])),
                                 camera_indices=None if ci is None else ci.reshape(-1, ci.shape[-1])[ri])
        if ray_bundle.times is not None:
            ray_samples.times = ray_bundle.times.reshape(-1, 1)[ri]
        self._prepass_payload = (s["feat"], s["corner_vals"]) if "feat" in s else None
        return ray_samples, ri, s["packed_info"]

    def _fused_ok(self) -> bool:
        return self.use_fused_render and not self.sampler.training and self.scene_aabb.is_cuda

    @torch.no_grad()
    def get_outputs_for_camera_ray_bundle(self, camera_ray_bundle: RayBundle) -> Dict[str, Tensor]:
        """nerfstudio Model.get_outputs_for_camera_ray_bundle (the eval entry point: evaluate_nersemble.py:143,
        util/render.py:39): chunk loop over eval_num_rays_per_chunk rays; tuple-wrapped per-sample outputs are skipped
        upstream, so the fused render's per-ray outputs are all that is needed -- no host synchronisation per chunk."""
        if not self._fused_ok():
            return super().get_outputs_for_camera_ray_bundle(camera_ray_bundle)
        n = self.config.eval_num_rays_per_chunk
        h, w = camera_ray_bundle.origins.shape[:2]
        # A camera frame has ONE timestep (evaluate_nersemble.py renders camera x timestep): when all rays carry the same
        # time (checked here: one host synchronisation per FRAME), the 32-member blend is hoisted out of the per-sample
        # path into a per-frame table (ops.NativeParams.frame_table) that every chunk of the frame gathers from L2.
        uniform_time = None
        if (self.frame_tables and camera_ray_bundle.times is not None and self.config.use_hash_ensemble
                and h * w >= self.frame_table_min_rays):
            t = camera_ray_bundle.times
            lo, hi = torch.stack([t.min(), t.max()]).tolist()
            uniform_time = lo if lo == hi else None
        lists: Dict[str, list] = {}
        for i in range(0, h * w, n):
            rb = camera_ray_bundle.get_row_major_sliced_ray_bundle(i, i + n)
            res = self._fused_render(rb, uniform_time)
            for name in ("rgb", "accumulation", "depth", "num_samples_per_ray", "deformation"):
                if name in res:
                    lists.setdefault(name, []).append(res[name])
        return {k: torch.cat(v).view(h, w, -1) for k, v in lists.items()}

    def get_outputs(self, ray_bundle: RayBundle, jitter: Optional[Tensor] = None):
        """models/nersemble_instant_ngp.py:280-364."""
        cfg = self.config
        wh, wd = self._windows()
        num_rays = len(ray_bundle)
        # the differentiable path is the TRAINING path (training-mode compositing); eval renders are inference-only
        needs_grad = self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if not needs_grad and self._fused_ok() and jitter is None:
            # eval: fused render; ONE host synchronisation (the packed sample count) to hand out exact-size per-sample tensors
            res = self._fused_render(ray_bundle)
            pk = res.packed()
            if pk["t_starts"].shape[0] > 0:
                ri = pk["ray_indices"].long()
                from ..nerfstudio_shim import Frustums
                o, d = ray_bundle.origins.reshape(-1, 3), ray_bundle.directions.reshape(-1, 3)
                origins = o[ri]
                ray_samples = RaySamples(frustums=Frustums(origins=origins, directions=d[ri], starts=pk["t_starts"][:, None],
                                                           ends=pk["t_ends"][:, None], pixel_area=torch.zeros_like(origins[:, :1])),
                                         camera_indices=None if ray_bundle.camera_indices is None else ray_bundle.camera_indices.reshape(-1, ray_bundle.camera_indices.shape[-1])[ri])
                if ray_bundle.times is not None:
                    ray_samples.times = ray_bundle.times.reshape(-1, 1)[ri]
                ray_samples.metadata = dict()
                outputs = {"rgb": res["rgb"], "accumulation": res["accumulation"], "depth": res["depth"],
                           "num_samples_per_ray": res["num_samples_per_ray"], "ray_samples": (ray_samples,),
                           "ray_indices": (ri,), "weights": (pk["weights"],)}
                if cfg.use_deformation_field:
                    ray_samples.frustums.set_offsets(pk["offsets"])
                    outputs["deformation"] = res["deformation"]
                return outputs
            # no sample at all: the reference inserts one fake sample (nersemble_volumetric_sampler.py:110-114) -> general path
        if self.use_fused_sampler and self.scene_aabb.is_cuda:
            ray_samples, ray_indices, packed_info = self._sample_packed(ray_bundle, jitter, want_payload=needs_grad)
        else:
            with torch.no_grad():
                ray_samples, ray_indices = self.sampler(
                    ray_bundle=ray_bundle, near_plane=cfg.near_plane, far_plane=cfg.far_plane,
                    render_step_size=cfg.render_step_size, alpha_thre=cfg.alpha_thre, cone_angle=cfg.cone_angle,
                    early_stop_eps=cfg.early_stop_eps, jitter=jitter)
            cnt = torch.zeros(num_rays, dtype=torch.long, device=ray_indices.device).index_add_(
                0, ray_indices, torch.ones_like(ray_indices))
            packed_info = torch.stack([cnt.cumsum(0) - cnt, cnt], -1)           # nerfacc.pack_info (:325)
        if ray_samples.metadata is None:
            ray_samples.metadata = dict()
        ray_times = self._ray_times(ray_bundle)
        starts = ray_samples.frustums.starts[..., 0].contiguous()
        ends = ray_samples.frustums.ends[..., 0].contiguous()
        if needs_grad:
            he = self.field.hash_ensemble
            params = [he.tables, self.field.mlp_base.params, self.field.mlp_head.params,
                                                               self.time_embedding.weight]
            if cfg.use_deformation_field:
                if not cfg.use_separate_deformation_time_embedding:
                    raise NotImplementedError("training with a shared time embedding (use_separate_deformation_time_embedding=False)")
                se3 = self.deformation_field.se3_field
                params.append(self.time_embedding_deformation.weight)
                for layer in se3.mlp_stem.layers:
                    params += [layer.weight, layer.bias]
                params += [se3.mlp_r.layers[0].weight, se3.mlp_r.layers[0].bias, se3.mlp_v.layers[0].weight, se3.mlp_v.layers[0].bias]
            res = _RenderFunction.apply(self, ray_bundle.origins, ray_bundle.directions, ray_times, starts, ends, ray_indices,
                                        packed_info, wh, wd, *params)
            rgb, acc, depth, weights = res[:4]
            outputs = {"rgb": rgb, "accumulation": acc, "depth": depth, "num_samples_per_ray": packed_info[:, 1],
                       "ray_samples": (ray_samples,), "ray_indices": (ray_indices,), "weights": (weights,)}
            if cfg.use_deformation_field:
                outputs["deformation"] = res[4]
                ray_samples.frustums.set_offsets(res[5])
            return outputs
        out = ops.render_packed(self.native_params(), ray_bundle.origins, ray_bundle.directions, ray_times, starts, ends,
                                ray_indices, packed_info, window_hash=wh, window_deform=wd,
                                use_deformation=cfg.use_deformation_field, training=self.training, **self._blend_opts())
        if cfg.use_deformation_field:
            ray_samples.frustums.set_offsets(out["offsets"])
        outputs = {
            "rgb": out["rgb"], "accumulation": out["accumulation"], "depth": out["depth"],
            "num_samples_per_ray": packed_info[:, 1],
            "ray_samples": (ray_samples,), "ray_indices": (ray_indices,), "weights": (out["weights"],),
        }
        if cfg.use_deformation_field:
            outputs["deformation"] = out["deformation"]
        return outputs

    def update_to_step(self, step: int) -> None:
        """nerfstudio Model.update_to_step: fast-forward the step-dependent schedules when a checkpoint is resumed
        (the reference relies on the BEFORE_TRAIN_ITERATION callbacks, which fire on the first resumed iteration)."""
        for sched in (self.sched_window_deform, self.sched_window_hash_encodings, self.sched_eps_depth):
            if sched is not None:
                sched.update(step)

    # ------------------------------------------------------------------ losses / metrics (models/base.py)
    def get_loss_dict(self, outputs, batch, metrics_dict=None) -> Dict[str, Tensor]:
        """models/nersemble_instant_ngp.py:366-407 -> models/base.py:90-249 (plain torch on per-ray/per-sample outputs)."""
        cfg = self.config
        if self.fused_losses and outputs["rgb"].is_cuda and "num_samples_per_ray" in outputs:
            return self._loss_dict_fused(outputs, batch)
        if self.sync_free_losses and outputs["rgb"].is_cuda:
            return self._loss_dict_sync_free(outputs, batch)
        ld: Dict[str, Tensor] = {}
        acc, depth = outputs["accumulation"], outputs["depth"]
        rs: RaySamples = outputs["ray_samples"][0]
        ri = outputs["ray_indices"][0]
        weights = outputs["weights"][0]
        rgb = outputs["rgb"]
        image = batch["image"].to(rgb.device)
        if cfg.use_masked_rgb_loss and "alpha_map" in batch:
            alpha_per_ray = batch["alpha_map"].squeeze(1).to(rgb.device) / 255.
            mask = alpha_per_ray > cfg.alpha_mask_threshold
            ld["rgb_loss"] = torch.nn.functional.mse_loss(image[mask], rgb[mask])
        else:
            ld["rgb_loss"] = torch.nn.functional.mse_loss(image, rgb)
        if cfg.lambda_alpha_loss is not None and cfg.lambda_alpha_loss > 0:
            alpha_per_ray = batch["alpha_map"].squeeze(1).to(rgb.device) / 255.
            bg = alpha_per_ray < 1
            if bg.any():
                ld["alpha_loss"] = (acc.squeeze(1)[bg] - alpha_per_ray[bg]).abs().mean() * cfg.lambda_alpha_loss
        starts = rs.frustums.starts.squeeze(1)
        ends = rs.frustums.ends.squeeze(1)
        if (cfg.lambda_empty_loss > 0 or cfg.lambda_near_loss > 0) and self.training:
            eps = self.sched_eps_depth.value
            tgt_ray = batch["depth_maps"].to(rgb.device)
            mid = (starts + ends) * 0.5
            tgt = tgt_ray[ri]
            w = weights.squeeze(1)
            if cfg.lambda_empty_loss > 0:
                vn = (tgt > 0) & (mid < tgt - eps)
                if vn.any():
                    ld["empty_loss"] = cfg.lambda_empty_loss * (w[vn] ** 2).mean()
            if cfg.lambda_near_loss > 0:
                near = (tgt > 0) & (tgt - eps <= mid) & (mid <= tgt + eps)
                expected = torch.distributions.Normal(0, (eps / 3) ** 2).cdf(mid - tgt)
                if near.any():
                    accumulated = _segment_exclusive_sum(w, ri, acc.shape[0]) + w
                    ld["near_loss"] = cfg.lambda_near_loss * ((accumulated[near] - expected[near]) ** 2).mean()
        if cfg.lambda_depth_loss > 0 and self.training:
            tgt_ray = batch["depth_maps"].to(rgb.device)
            dm = tgt_ray > 0
            if dm.any():
                ld["depth_loss"] = ((tgt_ray[dm] - depth.squeeze()[dm]) ** 2).mean() * cfg.lambda_depth_loss
        if cfg.lambda_dist_loss > 0:
            sel = ri < cfg.dist_loss_max_rays
            w = weights.squeeze(1)[sel]
            te_, ts_ = ends[sel], starts[sel]
            m, interval, rid = (te_ + ts_) * 0.5, te_ - ts_, ri[sel]
            if w.numel():
                n_rays = int(rid.max()) + 1
                w_pre = _segment_exclusive_sum(w, rid, n_rays)
                wm_pre = _segment_exclusive_sum(w * m, rid, n_rays)
                dist = ((1.0 / 3.0) * (interval * w * w).sum() + 2.0 * (w * (m * w_pre - wm_pre)).sum()) / n_rays
                ld["dist_loss"] = cfg.lambda_dist_loss * dist
        return ld

    def _loss_dict_fused(self, outputs, batch) -> Dict[str, Tensor]:
        """All six losses and their gradients in three kernel launches (csrc/nsb_losses.cu).  Same values as
        _loss_dict_sync_free (terms with an empty mask are present with value 0; fp32 scans instead of float64)."""
        cfg = self.config
        rgb = outputs["rgb"]
        dev = rgb.device
        rs: RaySamples = outputs["ray_samples"][0]
        cnt = outputs["num_samples_per_ray"].to(torch.int64)
        packed_info = torch.stack([cnt.cumsum(0) - cnt, cnt], -1)
        alpha = batch["alpha_map"].squeeze(1).to(dev) / 255. if "alpha_map" in batch else None
        train_terms = self.training and "depth_maps" in batch
        use = {"rgb_loss": True,
               "alpha_loss": bool(cfg.lambda_alpha_loss) and cfg.lambda_alpha_loss > 0 and alpha is not None,
               "empty_loss": train_terms and cfg.lambda_empty_loss > 0, "near_loss": train_terms and cfg.lambda_near_loss > 0,
               "depth_loss": train_terms and cfg.lambda_depth_loss > 0, "dist_loss": cfg.lambda_dist_loss > 0}
        lcfg = dict(use_masked_rgb=cfg.use_masked_rgb_loss, alpha_mask_threshold=cfg.alpha_mask_threshold,
                    lambda_alpha=cfg.lambda_alpha_loss if use["alpha_loss"] else 0.0,
                    lambda_empty=cfg.lambda_empty_loss if use["empty_loss"] else 0.0,
                    lambda_near=cfg.lambda_near_loss if use["near_loss"] else 0.0,
                    lambda_depth=cfg.lambda_depth_loss if use["depth_loss"] else 0.0,
                    lambda_dist=cfg.lambda_dist_loss if use["dist_loss"] else 0.0,
                    eps_depth=self.sched_eps_depth.value if self.sched_eps_depth is not None else 0.0,
                    dist_max_rays=cfg.dist_loss_max_rays)
        depth_target = batch["depth_maps"].to(dev) if (use["empty_loss"] or use["near_loss"] or use["depth_loss"]) else None
        vals = _FusedLosses.apply(rgb, outputs["accumulation"], outputs["depth"], outputs["weights"][0], packed_info,
                                  rs.frustums.starts, rs.frustums.ends, batch["image"].to(dev), alpha, depth_target, lcfg)
        return {name: vals[i] for i, name in enumerate(ops.LOSS_NAMES) if use[name]}

    def _loss_dict_sync_free(self, outputs, batch) -> Dict[str, Tensor]:
        """Same six losses (models/base.py:90-249) without device->host synchronisation: the reference selects
        elements with boolean indexing and `if mask.any()` (11 `nonzero` syncs per step, each draining
        the launch queue).  Here every masked mean is sum(mask * x) / count on the device.  Differences a caller can
        see: a term whose mask is empty is PRESENT with value 0 (the reference omits the key); values agree to
        summation order."""
        cfg = self.config
        ld: Dict[str, Tensor] = {}
        acc, depth = outputs["accumulation"], outputs["depth"]
        rs: RaySamples = outputs["ray_samples"][0]
        ri = outputs["ray_indices"][0]
        w = outputs["weights"][0].squeeze(1)
        rgb = outputs["rgb"]
        dev = rgb.device
        image = batch["image"].to(dev)
        n_rays = acc.shape[0]

        def masked_mean(x: Tensor, mask: Tensor, per_elem: int = 1) -> Tensor:
            cnt = mask.sum()
            # an empty mask gives 0 (x * mask sums to 0); the rgb loss keeps the reference's 0/0 = nan for an empty mask
            return (x * mask).sum() / (cnt.clamp(min=1) * per_elem)

        alpha_per_ray = batch["alpha_map"].squeeze(1).to(dev) / 255. if "alpha_map" in batch else None
        if cfg.use_masked_rgb_loss and alpha_per_ray is not None:
            mask = (alpha_per_ray > cfg.alpha_mask_threshold).to(rgb.dtype)
            ld["rgb_loss"] = (((image - rgb) ** 2) * mask[:, None]).sum() / (mask.sum() * 3)
        else:
            ld["rgb_loss"] = torch.nn.functional.mse_loss(image, rgb)
        if cfg.lambda_alpha_loss is not None and cfg.lambda_alpha_loss > 0:
            bg = (alpha_per_ray < 1).to(rgb.dtype)
            ld["alpha_loss"] = masked_mean((acc.squeeze(1) - alpha_per_ray).abs(), bg) * cfg.lambda_alpha_loss
        starts = rs.frustums.starts.squeeze(1)
        ends = rs.frustums.ends.squeeze(1)
        mid = (starts + ends) * 0.5
        if (cfg.lambda_empty_loss > 0 or cfg.lambda_near_loss > 0) and self.training:
            eps = self.sched_eps_depth.value
            tgt = batch["depth_maps"].to(dev)[ri]
            if cfg.lambda_empty_loss > 0:
                vn = ((tgt > 0) & (mid < tgt - eps)).to(w.dtype)
                ld["empty_loss"] = cfg.lambda_empty_loss * masked_mean(w ** 2, vn)
            if cfg.lambda_near_loss > 0:
                near = ((tgt > 0) & (tgt - eps <= mid) & (mid <= tgt + eps)).to(w.dtype)
                expected = torch.distributions.Normal(0, (eps / 3) ** 2).cdf(mid - tgt)
                accumulated = _segment_exclusive_sum(w, ri, n_rays) + w
                ld["near_loss"] = cfg.lambda_near_loss * masked_mean((accumulated - expected) ** 2, near)
        if cfg.lambda_depth_loss > 0 and self.training:
            tgt_ray = batch["depth_maps"].to(dev)
            dm = (tgt_ray > 0).to(rgb.dtype)
            ld["depth_loss"] = masked_mean((tgt_ray - depth.squeeze()) ** 2, dm) * cfg.lambda_depth_loss
        if cfg.lambda_dist_loss > 0:
            sel = (ri < cfg.dist_loss_max_rays).to(w.dtype)
            ws = w * sel                                           # rays beyond dist_loss_max_rays contribute nothing
            interval = ends - starts
            w_pre = _segment_exclusive_sum(ws, ri, n_rays)
            wm_pre = _segment_exclusive_sum(ws * mid, ri, n_rays)
            # torch_efficient_distloss divides by ray_id.max() + 1 of the selected samples (ray_indices are sorted)
            n_sel = (ri * (ri < cfg.dist_loss_max_rays)).max() + 1
            dist = ((1.0 / 3.0) * (interval * ws * ws).sum() + 2.0 * (ws * (mid * w_pre - wm_pre)).sum()) / n_sel
            ld["dist_loss"] = cfg.lambda_dist_loss * dist
        return ld

    def get_metrics_dict(self, outputs, batch) -> Dict[str, Tensor]:
        """models/nersemble_instant_ngp.py:409-422 (PSNR with data_range 1)."""
        rgb = outputs["rgb"]
        image = batch["image"].to(rgb.device)
        psnr = lambda a, b: -10.0 * torch.log10(torch.mean((a - b) ** 2))
        md = {"psnr": psnr(rgb, image), "num_samples_per_batch": outputs["num_samples_per_ray"].sum()}
        if "alpha_map" in batch:
            mask = batch["alpha_map"].squeeze(1).to(rgb.device) > 127
            md["psnr_masked"] = psnr(rgb[mask], image[mask])
        return md

    # ------------------------------------------------------------------ image metrics (evaluation)
    @staticmethod
    def _psnr(a: Tensor, b: Tensor) -> Tensor:
        """torchmetrics PeakSignalNoiseRatio(data_range=1.0)."""
        return -10.0 * torch.log10(torch.mean((a - b) ** 2))

    @staticmethod
    def _ssim(a: Tensor, b: Tensor, data_range: Optional[float] = None) -> Tensor:
        """torchmetrics.functional.structural_similarity_index_measure defaults: 11x11 gaussian window, sigma 1.5,
        k1 0.01, k2 0.03, reflect padding, mean over the image; data_range from the data when None.  a, b: [1,C,H,W]."""
        if data_range is None:
            data_range = float(max(a.max() - a.min(), b.max() - b.min()))
        c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
        k = torch.arange(11, dtype=a.dtype, device=a.device) - 5
        g = torch.exp(-(k / 1.5) ** 2 / 2); g = g / g.sum()
        C = a.shape[1]
        win = (g[:, None] * g[None, :]).expand(C, 1, 11, 11).contiguous()
        pad = lambda t: torch.nn.functional.pad(t, (5, 5, 5, 5), mode="reflect")
        conv = lambda t: torch.nn.functional.conv2d(pad(t), win, groups=C)
        mu_a, mu_b = conv(a), conv(b)
        s_aa, s_bb, s_ab = conv(a * a) - mu_a ** 2, conv(b * b) - mu_b ** 2, conv(a * b) - mu_a * mu_b
        ssim = ((2 * mu_a * mu_b + c1) * (2 * s_ab + c2)) / ((mu_a ** 2 + mu_b ** 2 + c1) * (s_aa + s_bb + c2))
        return ssim[..., 5:-5, 5:-5].mean() if min(ssim.shape[-2:]) > 10 else ssim.mean()

    @staticmethod
    def _colormap(x: Tensor, turbo: bool = False) -> Tensor:
        """[H,W,1] in [0,1] -> [H,W,3].  nerfstudio's colormaps when importable (matplotlib tables), else a
        dependency-free gradient (grey, or the polynomial turbo approximation) -- display only, no metric reads it."""
        try:
            from nerfstudio.utils import colormaps
            from nerfstudio.utils.colormaps import ColormapOptions
            return colormaps.apply_colormap(x, colormap_options=ColormapOptions(colormap="turbo")) if turbo else colormaps.apply_colormap(x)
        except Exception:  # noqa: BLE001
            x = torch.nan_to_num(x, 0.0).clamp(0, 1)
            if not turbo:
                return x.expand(*x.shape[:-1], 3)
            r = (0.1357 + x * (4.5974 - x * (42.3277 - x * (130.5887 - x * (150.5666 - x * 58.1375))))).clamp(0, 1)
            g = (0.0914 + x * (2.1856 + x * (4.8052 - x * (14.0195 - x * (4.2109 + x * 2.7747))))).clamp(0, 1)
            b = (0.1067 + x * (12.5925 - x * (60.1097 - x * (109.0745 - x * (88.5066 - x * 26.8183))))).clamp(0, 1)
            return torch.cat([r, g, b], -1)

    def get_image_metrics_and_images(self, outputs: Dict[str, Tensor], batch: Dict[str, Tensor]
                                     ) -> Tuple[Dict[str, float], Dict[str, Tensor]]:
        """models/nersemble_instant_ngp.py:424-500: full-image PSNR / SSIM / (LPIPS) / MSE, the masked variants, and the
        side-by-side images the trainer logs.  LPIPS needs pretrained network weights: `self.lpips` is an optional
        callable; without one the `lpips*` keys are NaN."""
        image = batch["image"].to(self.device)
        rgb = outputs["rgb"]
        acc_img = self._colormap(outputs["accumulation"])
        depth = outputs["depth"]
        near, far = float(torch.min(depth)), float(torch.max(depth))      # apply_depth_colormap: normalise, turbo, white where acc = 0
        depth_img = self._colormap(((depth - near) / (far - near + 1e-10)).clamp(0, 1), turbo=True)
        depth_img = depth_img * outputs["accumulation"] + (1 - outputs["accumulation"])
        error_img = self._colormap(((rgb - image) ** 2).mean(dim=-1, keepdim=True), turbo=True)
        images_dict = {"img": torch.cat([image, rgb], dim=1), "accumulation": acc_img, "depth": depth_img, "error": error_img}
        im, rg = torch.moveaxis(image, -1, 0)[None], torch.moveaxis(rgb, -1, 0)[None]
        lp = (lambda a, b: float(self.lpips(a, b))) if self.lpips is not None else (lambda a, b: float("nan"))
        metrics_dict = {"psnr": float(self._psnr(im, rg)), "ssim": float(self._ssim(im, rg)), "lpips": lp(im, rg),
                        "mse": float(torch.nn.functional.mse_loss(im, rg)), "cam_id": float(batch["cam_ids"])}
        if "deformation" in outputs:
            d = outputs["deformation"]                      # scene-flow colouring: direction -> colour, magnitude -> saturation
            mag = d.norm(dim=-1, keepdim=True)
            images_dict["deformation"] = (0.5 + 0.5 * d / (mag.max() + 1e-10)).clamp(0, 1)
        if "alpha_map" in batch:
            am = torch.as_tensor(batch["alpha_map"]).to(rgb) / 255.
            image_m = am * image + (1 - am)
            rgb_m = am * rgb + (1 - am)
            images_dict["img_masked"] = torch.cat([image_m, rgb_m], dim=1)
            im_m, rg_m = torch.moveaxis(image_m, -1, 0)[None], torch.moveaxis(rgb_m, -1, 0)[None]
            metrics_dict.update(psnr_masked=float(self._psnr(im_m, rg_m)), ssim_masked=float(self._ssim(im_m, rg_m)),
                                lpips_masked=lp(im_m, rg_m), mse_masked=float(torch.nn.functional.mse_loss(im_m, rg_m)))
        return metrics_dict, images_dict

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        """models/nersemble_instant_ngp.py:502-514."""
        groups = {"fields": list(self.field.parameters())}
        if self.time_embedding is not None:
            groups["embeddings"] = list(self.time_embedding.parameters())
            if self.config.use_separate_deformation_time_embedding:
                groups["embeddings"].extend(list(self.time_embedding_deformation.parameters()))
        if self.config.use_deformation_field:
            groups["deformation_field"] = list(self.deformation_field.parameters())
        return groups
