"""CPU restatement of the nerfstudio 0.3.1 pieces the reference's hot path uses  [3P-mem].

TEST INFRASTRUCTURE (see oracle/__init__.py).  nerfstudio==0.3.1 (environment.yml:29) is
not installed / not on disk.  Restated here (minimal, duck-typed):
  cameras.rays.{Frustums,RaySamples,RayBundle}, data.scene_box.SceneBox,
  field_components.mlp.MLP, field_components.encodings.NeRFEncoding,
  field_components.activations.trunc_exp, fields.base_field.shift_directions_for_tcnn,
  model_components.renderers.{RGBRenderer,DepthRenderer,AccumulationRenderer},
  model_components.ray_samplers.VolumetricSampler, models.base_model.{Model,ModelConfig},
  models.instant_ngp.{NGPModel,InstantNGPModelConfig}, engine.callbacks.*
Reference call sites are listed in SURVEY.md 8(c).  PARITY UNPINNED for this layer.

Upstream map (nerfstudio v0.3.1, nerfstudio-project/nerfstudio):
  Frustums / RaySamples / RayBundle   nerfstudio/cameras/rays.py (get_positions = o + d*(s+e)/2 [+ offsets], set_offsets,
                                      get_row_major_sliced_ray_bundle)
  SceneBox                            nerfstudio/data/scene_box.py: get_normalized_positions ((p - aabb[0]) / (aabb[1] - aabb[0]))
  MLP                                 nerfstudio/field_components/mlp.py: MLP.build_nn_modules / forward (skip: cat([in_tensor, x]))
  NeRFEncoding, expected_sin          nerfstudio/field_components/encodings.py, nerfstudio/utils/math.py
  _TruncExp / trunc_exp               nerfstudio/field_components/activations.py (bwd: g * exp(clamp(x, -15, 15)))
  shift_directions_for_tcnn           nerfstudio/fields/base_field.py
  FieldHeadNames                      nerfstudio/field_components/field_heads.py
  RGBRenderer / AccumulationRenderer / DepthRenderer   nerfstudio/model_components/renderers.py (combine_rgb, blend_background,
                                      eval-mode nan_to_num + clamp_; 'expected' depth with global clip to steps.min/max)
  VolumetricSampler                   nerfstudio/model_components/ray_samplers.py: VolumetricSampler.get_sigma_fn
  TrainingCallback*                   nerfstudio/engine/callbacks.py
  Model / ModelConfig                 nerfstudio/models/base_model.py
  NGPModel / InstantNGPModelConfig    nerfstudio/models/instant_ngp.py
"""
from __future__ import annotations

from dataclasses import dataclass, field
from enum import Enum, auto
from typing import Any, Callable, Dict, List, Optional, Tuple, Type

import torch
from torch import nn

from . import nerfacc_cpu as nerfacc


# ------------------------------------------------------------------ cameras.rays
class _TensorBag:
    """Tiny stand-in for nerfstudio's TensorDataclass: holds tensors with a common leading shape."""

    def __len__(self):
        return self.shape[0]


class Frustums(_TensorBag):
    def __init__(self, origins, directions, starts, ends, pixel_area, offsets=None):
        self.origins = origins
        self.directions = directions
        self.starts = starts
        self.ends = ends
        self.pixel_area = pixel_area
        self.offsets = offsets

    @property
    def shape(self):
        return self.origins.shape[:-1]

    def get_positions(self) -> torch.Tensor:
        pos = self.origins + self.directions * (self.starts + self.ends) / 2
        if self.offsets is not None:
            pos = pos + self.offsets
        return pos

    def set_offsets(self, offsets):
        self.offsets = offsets


class RaySamples(_TensorBag):
    def __init__(self, frustums: Frustums, camera_indices=None, deltas=None, spacing_starts=None,
                 spacing_ends=None, spacing_to_euclidean_fn=None, metadata=None, times=None):
        self.frustums = frustums
        self.camera_indices = camera_indices
        self.deltas = deltas
        self.metadata = metadata
        self.times = times

    @property
    def shape(self):
        return self.frustums.shape


class RayBundle(_TensorBag):
    def __init__(self, origins, directions, pixel_area=None, camera_indices=None, nears=None, fars=None,
                 metadata=None, times=None):
        self.origins = origins
        self.directions = directions
        self.pixel_area = pixel_area
        self.camera_indices = camera_indices
        self.nears = nears
        self.fars = fars
        self.metadata = metadata if metadata is not None else {}
        self.times = times

    @property
    def shape(self):
        return self.origins.shape[:-1]

    def get_row_major_sliced_ray_bundle(self, start, end):
        def sl(t):
            return None if t is None else t.reshape(-1, t.shape[-1])[start:end]
        return RayBundle(sl(self.origins), sl(self.directions), sl(self.pixel_area), sl(self.camera_indices),
                         sl(self.nears), sl(self.fars), {k: sl(v) for k, v in self.metadata.items()},
                         sl(self.times))


# ------------------------------------------------------------------ data.scene_box
class SceneBox:
    def __init__(self, aabb: torch.Tensor):
        self.aabb = aabb

    @staticmethod
    def get_normalized_positions(positions, aabb):
        aabb_lengths = aabb[1] - aabb[0]
        return (positions - aabb[0]) / aabb_lengths


# ------------------------------------------------------------------ field_components
class MLP(nn.Module):
    """field_components/mlp.py: Linear layers WITH bias; skip concatenates [input, hidden]."""

    def __init__(self, in_dim, num_layers, layer_width, out_dim=None, skip_connections=None,
                 activation=nn.ReLU(), out_activation=None):
        super().__init__()
        self.in_dim = in_dim
        self.out_dim = out_dim if out_dim is not None else layer_width
        self.num_layers = num_layers
        self.layer_width = layer_width
        self.skip_connections = skip_connections
        self._skip_connections = set(skip_connections) if skip_connections else set()
        self.activation = activation
        self.out_activation = out_activation
        layers = []
        if num_layers == 1:
            layers.append(nn.Linear(in_dim, self.out_dim))
        else:
            for i in range(num_layers - 1):
                if i == 0:
                    assert i not in self._skip_connections
                    layers.append(nn.Linear(in_dim, layer_width))
                elif i in self._skip_connections:
                    layers.append(nn.Linear(layer_width + in_dim, layer_width))
                else:
                    layers.append(nn.Linear(layer_width, layer_width))
            layers.append(nn.Linear(layer_width, self.out_dim))
        self.layers = nn.ModuleList(layers)

    @staticmethod
    def _lin(layer, x):
        """nn.Linear under the active precision emulation: "reference"+autocast = fp16 operands
        and fp16 output (torch.autocast in engine/nersemble_trainer.py:182; eval and the
        occupancy callback run WITHOUT autocast -> fp32); "kernel" = fp16 operands, fp32
        accumulate and bias (the CUDA kernel)."""
        from .tcnn_cpu import Precision, half_round
        if Precision.mode == "kernel":
            return half_round(x) @ half_round(layer.weight).t() + layer.bias
        if Precision.mode == "reference" and Precision.autocast:
            return half_round(half_round(x) @ half_round(layer.weight).t() + half_round(layer.bias))
        return layer(x)

    def forward(self, in_tensor):
        from .tcnn_cpu import Precision, half_round
        x = in_tensor
        for i, layer in enumerate(self.layers):
            if i in self._skip_connections:
                x = torch.cat([in_tensor, x], -1)
            x = self._lin(layer, x)
            if self.activation is not None and i < len(self.layers) - 1:
                x = self.activation(x)
                if Precision.mode == "kernel":
                    x = half_round(x)
        if self.out_activation is not None:
            x = self.out_activation(x)
            if Precision.mode == "kernel":
                x = half_round(x)
        return x


class NeRFEncoding(nn.Module):
    def __init__(self, in_dim, num_frequencies, min_freq_exp, max_freq_exp, include_input=False):
        super().__init__()
        self.in_dim = in_dim
        self.num_frequencies = num_frequencies
        self.min_freq = min_freq_exp
        self.max_freq = max_freq_exp
        self.include_input = include_input

    def get_out_dim(self) -> int:
        out_dim = self.in_dim * self.num_frequencies * 2
        if self.include_input:
            out_dim += self.in_dim
        return out_dim


def expected_sin(x_means, x_vars):
    return torch.exp(-0.5 * x_vars) * torch.sin(x_means)


class _TruncExp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        x = ctx.saved_tensors[0]
        return g * torch.exp(x.clamp(-15, 15))


trunc_exp = _TruncExp.apply


def shift_directions_for_tcnn(directions):
    return (directions + 1.0) / 2.0


class FieldHeadNames(Enum):
    RGB = "rgb"
    SH = "sh"
    DENSITY = "density"
    NORMALS = "normals"
    PRED_NORMALS = "pred_normals"
    UNCERTAINTY = "uncertainty"
    TRANSIENT_RGB = "transient_rgb"
    TRANSIENT_DENSITY = "transient_density"
    SEMANTICS = "semantics"


class Field(nn.Module):
    pass


class TCNNNerfactoField(Field):
    pass


# ------------------------------------------------------------------ renderers
class RGBRenderer(nn.Module):
    """model_components/renderers.py: packed path accumulates with nerfacc; background blended as
    rgb + bg*(1-acc); eval: nan_to_num before, clamp_(0,1) after."""

    def __init__(self, background_color="random"):
        super().__init__()
        self.background_color = background_color

    def forward(self, rgb, weights, ray_indices=None, num_rays=None):
        if not self.training:
            rgb = torch.nan_to_num(rgb)
        comp = nerfacc.accumulate_along_rays(weights[..., 0], values=rgb, ray_indices=ray_indices, n_rays=num_rays)
        acc = nerfacc.accumulate_along_rays(weights[..., 0], values=None, ray_indices=ray_indices, n_rays=num_rays)
        assert self.background_color == "white"
        bg = torch.ones(3, dtype=comp.dtype)
        comp = comp + bg * (1.0 - acc)
        if not self.training:
            comp = torch.clamp(comp, min=0.0, max=1.0)
        return comp


class AccumulationRenderer(nn.Module):
    def forward(self, weights, ray_indices=None, num_rays=None):
        return nerfacc.accumulate_along_rays(weights[..., 0], values=None, ray_indices=ray_indices, n_rays=num_rays)


class DepthRenderer(nn.Module):
    def __init__(self, method="median"):
        super().__init__()
        self.method = method

    def forward(self, weights, ray_samples, ray_indices=None, num_rays=None):
        assert self.method == "expected"
        eps = 1e-10
        steps = (ray_samples.frustums.starts + ray_samples.frustums.ends) / 2
        depth = nerfacc.accumulate_along_rays(weights[..., 0], values=steps, ray_indices=ray_indices, n_rays=num_rays)
        accumulation = nerfacc.accumulate_along_rays(weights[..., 0], values=None, ray_indices=ray_indices,
                                                     n_rays=num_rays)
        depth = depth / (accumulation + eps)
        depth = torch.clip(depth, steps.min(), steps.max())
        return depth


# ------------------------------------------------------------------ samplers
DensityFn = Callable


class VolumetricSampler(nn.Module):
    def __init__(self, occupancy_grid, density_fn=None):
        super().__init__()
        assert occupancy_grid is not None
        self.density_fn = density_fn
        self.occupancy_grid = occupancy_grid

    def get_sigma_fn(self, origins, directions, times=None):
        if self.density_fn is None or not self.training:
            return None
        density_fn = self.density_fn

        def sigma_fn(t_starts, t_ends, ray_indices):
            t_origins = origins[ray_indices]
            t_dirs = directions[ray_indices]
            positions = t_origins + t_dirs * (t_starts + t_ends)[:, None] / 2.0
            if times is None:
                return density_fn(positions).squeeze(-1)
            return density_fn(positions, times[ray_indices]).squeeze(-1)

        return sigma_fn


# ------------------------------------------------------------------ engine.callbacks
class TrainingCallbackLocation(Enum):
    BEFORE_TRAIN_ITERATION = auto()
    AFTER_TRAIN_ITERATION = auto()


@dataclass
class TrainingCallbackAttributes:
    optimizers: Any = None
    grad_scaler: Any = None
    pipeline: Any = None


class TrainingCallback:
    def __init__(self, where_to_run, func, update_every_num_iters=None, iters=None, args=None, kwargs=None):
        self.where_to_run = where_to_run
        self.update_every_num_iters = update_every_num_iters
        self.iters = iters
        self.func = func
        self.args = args if args is not None else []
        self.kwargs = kwargs if kwargs is not None else {}

    def run_callback(self, step: int):
        if self.update_every_num_iters is not None:
            if step % self.update_every_num_iters == 0:
                self.func(*self.args, **self.kwargs, step=step)
        elif self.iters is not None and step in self.iters:
            self.func(*self.args, **self.kwargs, step=step)

    def run_callback_at_location(self, step, location):
        if location in self.where_to_run:
            self.run_callback(step)


# ------------------------------------------------------------------ models
@dataclass
class ModelConfig:
    _target: Type = field(default_factory=lambda: Model)
    enable_collider: bool = True
    collider_params: Optional[Dict[str, float]] = None
    loss_coefficients: Optional[Dict[str, float]] = None
    eval_num_rays_per_chunk: int = 4096

    def setup(self, **kwargs):
        return self._target(self, **kwargs)


class Model(nn.Module):
    def __init__(self, config, scene_box, num_train_data, **kwargs):
        super().__init__()
        self.config = config
        self.scene_box = scene_box
        self.num_train_data = num_train_data
        self.kwargs = kwargs
        self.collider = None
        self.populate_modules()
        self.device_indicator_param = nn.Parameter(torch.empty(0))

    @property
    def device(self):
        return self.device_indicator_param.device

    def populate_modules(self):
        pass

    def get_training_callbacks(self, training_callback_attributes) -> List[TrainingCallback]:
        return []

    def forward(self, ray_bundle):
        return self.get_outputs(ray_bundle)

    @torch.no_grad()
    def get_outputs_for_camera_ray_bundle(self, camera_ray_bundle) -> Dict[str, torch.Tensor]:
        num_rays_per_chunk = self.config.eval_num_rays_per_chunk
        image_height, image_width = camera_ray_bundle.origins.shape[:2]
        num_rays = image_height * image_width
        outputs_lists: Dict[str, list] = {}
        for i in range(0, num_rays, num_rays_per_chunk):
            ray_bundle = camera_ray_bundle.get_row_major_sliced_ray_bundle(i, i + num_rays_per_chunk)
            outputs = self.forward(ray_bundle=ray_bundle)
            for name, out in outputs.items():
                if not torch.is_tensor(out):
                    continue
                outputs_lists.setdefault(name, []).append(out)
        return {k: torch.cat(v).view(image_height, image_width, -1) for k, v in outputs_lists.items()}


@dataclass
class InstantNGPModelConfig(ModelConfig):
    """models/instant_ngp.py defaults (all overridden by train_nersemble.py:186-197 anyway)."""
    _target: Type = field(default_factory=lambda: NGPModel)
    enable_collider: bool = False
    collider_params: Optional[Dict[str, float]] = None
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


class NGPModel(Model):
    def get_param_groups(self):
        if self.field is None:
            raise ValueError("populate_fields() must be called before get_param_groups")
        return {"fields": list(self.field.parameters())}


class MSELoss(nn.MSELoss):
    pass
