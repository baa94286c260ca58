"""NeRSembleNeRFactoField -- mirror of fields/nersemble_nerfacto_field.py:30-402 (hash-ensemble configuration)."""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
from torch import Tensor, nn
from torch.autograd.function import once_differentiable

from .. import ops, packing
from ..nerfstudio_shim import FieldHeadNames, Frustums, RaySamples
from .components import HashEnsemble, HashEnsembleConfig, _FlatParams, _needs_grad

BASE_SHAPES = [(64, 32), (16, 64)]                 # tcnn mlp_base: 32 -> 64 -> 16 (1 + 15 geo feats)
HEAD_SHAPES = [(64, 32), (64, 64), (16, 64)]       # tcnn mlp_head: 18 (pad 32 with 1.0) -> 64 -> 64 -> 3 (pad 16)


class _FieldFunction(torch.autograd.Function):
    """density_fn / forward of the field with gradients for mlp_base.params, mlp_head.params, the hash tables (dense
    fp32 `.grad`), the per-sample time codes and the positions: nsb_field_forward (saving the blended features and the
    normalised positions) / nsb_field_backward.  Returns (sigma [n], rgb [n,3] or None)."""

    @staticmethod
    def forward(ctx, field, positions, directions, time_codes, window, want_rgb, base_params, head_params, tables):
        P = field._native_params()
        want = ("sigma", "rgb") if want_rgb else ("sigma",)
        out = ops.field_forward(P, window_hash=window, use_deformation=False, positions=positions,
                                sample_directions=directions, sample_blend_codes=time_codes, want=want + ("feat", "xs"),
                                **field._opts())
        ctx.field, ctx.P, ctx.window = field, P, window
        ctx.saved = {k: out.get(k) for k in ("feat", "xs", "sigma", "rgb")}    # rgb: None for the density alone
        ctx.save_for_backward(positions, directions, time_codes)
        if want_rgb:
            return out["sigma"], out["rgb"]
        return out["sigma"], None

    @staticmethod
    @once_differentiable
    def backward(ctx, g_sigma, g_rgb):
        positions, directions, time_codes = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = ops.field_backward(ctx.P, ctx.saved, g_sigma, g_rgb, window_hash=ctx.window,
                               loss_scale=float(ctx.field.mlp_loss_scale), want_tables=need[8], want_codes=need[3],
                               want_dx=need[1], rank1=False, positions=positions, sample_directions=directions,
                               sample_blend_codes=time_codes, **ctx.field._opts())
        d_pos = None
        if need[1]:     # dL/d(world position) = dL/d(normalised position) / aabb size; 0 outside the box (kernel selector)
            aabb = ctx.field.aabb.detach().float()
            d_pos = g["d_xs"] / (aabb[1] - aabb[0])
        return (None, d_pos, None, g.get("d_sample_blend_codes"), None, None, g["d_base_w"], g["d_head_w"],
                g.get("d_tables"))


def _xavier_flat(shapes, gen):
    parts = []
    for (o, i) in shapes:
        b = math.sqrt(6.0 / (i + o))
        parts.append((torch.rand(o * i, generator=gen) * 2 - 1) * b)
    return torch.cat(parts)


class NeRSembleNeRFactoField(nn.Module):
    """Constructor keeps the reference's keyword surface (nersemble_nerfacto_field.py:32-62); options the
    NeRSemble recipe never enables (transient / semantics / normals / appearance embedding / scene contraction /
    SH directions) are rejected instead of silently ignored."""

    def __init__(self, aabb: Tensor, num_images: int, num_layers: int = 2, hidden_dim: int = 64, geo_feat_dim: int = 15,
                 num_levels: int = 16, max_res: int = 2048, log2_hashmap_size: int = 19, num_layers_color: int = 3,
                 num_layers_transient: int = 2, hidden_dim_color: int = 64, hidden_dim_transient: int = 64,
                 appearance_embedding_dim: int = 32, transient_embedding_dim: int = 16,
                 use_transient_embedding: bool = False, use_semantics: bool = False, num_semantic_classes: int = 100,
                 pass_semantic_gradients: bool = False, use_pred_normals: bool = False,
                 use_average_appearance_embedding: bool = False, spatial_distortion=None,
                 use_appearance_embedding: bool = False, spherical_harmonics_degree: int = 4,
                 use_hash_ensemble: bool = False, hash_ensemble_config: Optional[HashEnsembleConfig] = None,
                 max_n_samples_per_batch: int = -1, seed: Optional[int] = None) -> None:
        super().__init__()
        unsupported = dict(use_transient_embedding=use_transient_embedding, use_semantics=use_semantics,
                           use_pred_normals=use_pred_normals, use_appearance_embedding=use_appearance_embedding)
        bad = [k for k, v in unsupported.items() if v]
        if bad or spatial_distortion is not None or spherical_harmonics_degree != 0 or not use_hash_ensemble:
            raise NotImplementedError(
                f"the CUDA field supports the NeRSemble recipe only (train_nersemble.py:184-240): hash ensemble, "
                f"identity direction encoding, no scene contraction; got {bad}, sh_degree={spherical_harmonics_degree}")
        assert num_layers == 2 and hidden_dim == 64 and geo_feat_dim == 15 and num_layers_color == 3 and hidden_dim_color == 64
        self.register_buffer("aabb", aabb)
        self.geo_feat_dim = geo_feat_dim
        self.register_buffer("max_res", torch.tensor(max_res))
        self.register_buffer("num_levels", torch.tensor(num_levels))
        self.register_buffer("log2_hashmap_size", torch.tensor(log2_hashmap_size))
        self.num_images = num_images
        self.use_hash_ensemble = True
        self.max_n_samples_per_batch = max_n_samples_per_batch
        # empty tcnn modules kept for state_dict / param-group compatibility (Identity direction encoding,
        # unused Frequency position encoding: nersemble_nerfacto_field.py:106-112,132-135)
        self.direction_encoding = _FlatParams(torch.zeros(0))
        self.hash_ensemble = HashEnsemble(hash_ensemble_config, seed=seed)
        self.position_encoding = _FlatParams(torch.zeros(0))
        g = torch.Generator()
        if seed is not None:
            g.manual_seed(seed + 1)
        self.mlp_base = _FlatParams(_xavier_flat(BASE_SHAPES, g))
        self.mlp_head = _FlatParams(_xavier_flat(HEAD_SHAPES, g))
        self.mlp_loss_scale = 128.0      # the backward's fp16 MLP deltas are scaled by this and the gradients divided back
        self._native = None
        self._native_version = None

    # ---- parameter views
    def base_weights(self):
        return packing.split_tcnn_mlp_params(self.mlp_base.params, BASE_SHAPES)

    def head_weights(self):
        return packing.split_tcnn_mlp_params(self.mlp_head.params, HEAD_SHAPES)

    def _native_params(self) -> ops.NativeParams:
        v = (self.mlp_base.params._version, self.mlp_head.params._version, self.mlp_base.params.data_ptr())
        if self._native is None or v != self._native_version:
            with torch.no_grad():
                self._native = ops.NativeParams.build(tables=None, time_emb=None, aabb=self.aabb, levels=self.hash_ensemble.levels,
                                                      base_w=self.base_weights(), head_w=self.head_weights(),
                                                      device=self.aabb.device)
            self._native_version = v
        self._native.tables = self.hash_ensemble.native_tables()
        return self._native

    def _opts(self):
        he = self.hash_ensemble
        return dict(disable_initial=he.disable_initial_hash_ensemble, soft_transition=he.use_soft_transition)

    def _grad_params(self):
        """The parameters _FieldFunction returns gradients for, in its input order."""
        return [self.mlp_base.params, self.mlp_head.params, self.hash_ensemble.tables]

    # ---- reference API
    def density_fn(self, positions: Tensor, times: Optional[Tensor] = None, window_hash_encodings: Optional[float] = None,
                   time_codes: Optional[Tensor] = None) -> Tensor:
        """nersemble_nerfacto_field.py:228-248."""
        if _needs_grad(positions, time_codes, *self._grad_params()):
            sigma, _ = _FieldFunction.apply(self, positions, None, time_codes, window_hash_encodings, False,
                                            *self._grad_params())
            return sigma[:, None]
        out = ops.field_forward(self._native_params(), window_hash=window_hash_encodings, use_deformation=False,
                                positions=positions, sample_blend_codes=time_codes, want=("sigma",), **self._opts())
        return out["sigma"][:, None]

    def get_density(self, ray_samples: RaySamples, window_hash_encodings: float) -> Tuple[Tensor, Optional[Tensor]]:
        """nersemble_nerfacto_field.py:250-301.  The geometry features stay inside the fused kernel, so the second
        element is None; use forward() for colours."""
        tc = ray_samples.metadata["time_codes"]
        return self.density_fn(ray_samples.frustums.get_positions(), None, window_hash_encodings, tc), None

    def get_outputs(self, ray_samples: RaySamples, density_embedding: Optional[Tensor] = None):
        raise NotImplementedError("density and colour MLPs are fused: call forward(ray_samples, ...) (nsb_field_forward)")

    def forward(self, ray_samples: RaySamples, compute_normals: bool = False,
                window_hash_encodings: Optional[float] = None) -> Dict[FieldHeadNames, Tensor]:
        """nersemble_nerfacto_field.py:385-402."""
        if compute_normals:
            raise NotImplementedError("compute_normals")
        if ray_samples.camera_indices is None:
            raise AttributeError("Camera indices are not provided.")
        tc = ray_samples.metadata["time_codes"]
        pos = ray_samples.frustums.get_positions()
        if _needs_grad(pos, tc, *self._grad_params()):
            sigma, rgb = _FieldFunction.apply(self, pos, ray_samples.frustums.directions, tc, window_hash_encodings, True,
                                              *self._grad_params())
            return {FieldHeadNames.RGB: rgb, FieldHeadNames.DENSITY: sigma[:, None]}
        out = ops.field_forward(self._native_params(), window_hash=window_hash_encodings, use_deformation=False,
                                positions=pos, sample_directions=ray_samples.frustums.directions, sample_blend_codes=tc,
                                want=("sigma", "rgb"), **self._opts())
        return {FieldHeadNames.RGB: out["rgb"], FieldHeadNames.DENSITY: out["sigma"][:, None]}
