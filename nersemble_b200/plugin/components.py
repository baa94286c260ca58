"""HashEnsemble, SE3DeformationField, GenericScheduler -- mirrors of
field_components/hash_ensemble.py, field_components/deformation_field.py and
engine/generic_scheduler.py of the reference, computing through libnsb."""
from __future__ import annotations

import math
import weakref
from dataclasses import dataclass
from math import ceil
from typing import Dict, List, Literal, Optional, Tuple

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from .. import ops, packing


def _needs_grad(*tensors) -> bool:
    """True when autograd has to record the call; otherwise the component runs its forward-only path."""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


class _HashEnsembleFunction(torch.autograd.Function):
    """HashEnsemble.forward with gradients for the tables (dense fp32 `.grad`), the conditioning code and the input
    position: nsb_hash_blend_forward / nsb_hash_blend_backward."""

    @staticmethod
    def forward(ctx, he, in_tensor, conditioning_code, tables, window):
        P = he._blend_params()
        out = ops.hash_blend_forward(P, in_tensor, conditioning_code, window_hash=window, out_half=True, **he._blend_opts())
        ctx.he, ctx.P, ctx.window = he, P, window
        ctx.save_for_backward(in_tensor, conditioning_code)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        x, code = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = ops.hash_blend_backward(ctx.P, x, code, g_out, window_hash=ctx.window, want_tables=need[3],
                                    want_codes=need[2], want_dx=need[1], **ctx.he._blend_opts())
        return (None, g.get("d_x"), g.get("d_codes"), g.get("d_tables"), None)


class GenericScheduler(nn.Module):
    """engine/generic_scheduler.py:4-30 (same attribute semantics: the model reads `.value`)."""

    def __init__(self, init_value, final_value, begin_step, end_step) -> None:
        super().__init__()
        self.init_value, self.final_value = init_value, final_value
        self.begin_step, self.end_step = begin_step, end_step
        self.value = final_value

    def update(self, step):
        if step > self.end_step:
            self.value = self.final_value
        elif step < self.begin_step:
            self.value = self.init_value
        else:
            delta = min(max((step - self.begin_step) / (self.end_step - self.begin_step), 0), 1) * (
                self.final_value - self.init_value)
            self.value = self.init_value + delta

    def get_value(self):
        return self.value if self.training else self.final_value


class _FlatParams(nn.Module):
    """Holds one flat fp32 `.params` tensor like a tcnn module, so state_dict keys match the reference
    (`...hash_encodings.{c}.params`, `field.mlp_base.params`, `field.mlp_head.params`)."""

    def __init__(self, init: torch.Tensor):
        super().__init__()
        self.params = nn.Parameter(init)


@dataclass
class TCNNHashEncodingConfig:
    """hash_ensemble.py:31-39."""
    n_dims_to_encode: int = 3
    n_levels: int = 16
    n_features_per_level: int = 2
    log2_hashmap_size: int = 19
    base_resolution: int = 16
    per_level_scale: float = 1.4472692012786865
    interpolation: Literal['Linear', 'Nearest', 'Smoothstep'] = 'Linear'

    def level_table(self):
        return packing.level_table(self.n_levels, self.log2_hashmap_size, self.base_resolution, self.per_level_scale)


@dataclass
class HashEnsembleConfig:
    """hash_ensemble.py:55-66."""
    n_hash_encodings: int
    hash_encoding_config: TCNNHashEncodingConfig
    disable_initial_hash_ensemble: bool = False
    use_soft_transition: bool = False


class _GridView:
    """Read/write shim with the reference's `hash_encodings[c].params` spelling.  `.params` is a copy of grid c in tcnn's
    flat layout; the storage is HashEnsemble.tables (native layout)."""

    def __init__(self, owner: "HashEnsemble", c: int):
        self._owner, self._c = owner, c

    @property
    def params(self) -> torch.Tensor:
        t = self._owner.tables.detach()
        return t[:, 4 * self._c:4 * self._c + 4, :].reshape(-1)


class HashEnsemble(nn.Module):
    """hash_ensemble.py:69-168.

    Storage.  The reference holds 8 tcnn grids of 8 features/level (`hash_encodings.{c}.params`, flat fp32).  Here the
    ONE trainable tensor is `tables`, fp32 [total_entries, 32 members, 2 feats] -- the layout the kernels gather (one
    128-byte fp16 line per entry) and scatter gradients into, so a training step never permutes 1.6 GB between
    layouts (index/cat/copy glue every step).  state_dict()/load_state_dict() still speak the
    reference's keys and flat shapes (hooks below), and the parameter sits in the same `fields` group.  The fp16 copy
    the forward kernels read is a cache refreshed when `tables` changes (or written by the fused optimiser)."""

    def __init__(self, config: HashEnsembleConfig, seed: Optional[int] = None):
        super().__init__()
        hc = config.hash_encoding_config
        assert config.n_hash_encodings == 32 and hc.n_features_per_level == 2 and hc.n_levels == 16 \
            and hc.n_dims_to_encode == 3 and hc.interpolation == 'Linear', \
            "the CUDA kernels are specialised for the reference configuration: 32 x (16 levels, 2 features), Linear"
        self.n_hash_encodings = config.n_hash_encodings
        self.hash_encoding_config = hc
        self.disable_initial_hash_ensemble = config.disable_initial_hash_ensemble
        self.use_soft_transition = config.use_soft_transition
        n_total_features = config.n_hash_encodings * hc.n_features_per_level
        self.levels = hc.level_table()
        self.n_grids = ceil(n_total_features / 8)
        g = torch.Generator()
        if seed is not None:
            g.manual_seed(seed)
        # tcnn grid init U(-1e-4, 1e-4), drawn grid by grid like the reference builds its ModuleList
        grids = [(torch.rand(self.levels["total_entries"] * 8, generator=g) * 2 - 1) * 1e-4 for _ in range(self.n_grids)]
        self.tables = nn.Parameter(packing.tables_from_tcnn(grids))
        del grids
        self.n_output_dims = hc.n_levels * hc.n_features_per_level
        self._native = None
        self._native_version = None
        self._shadow = None
        # fused optimiser protocol (nersemble_b200/optim.py): with defer_table_grad the training backward parks the
        # table gradient here in rank-1 form instead of writing a dense `.grad`
        self.defer_table_grad = False
        self.pending_table_grad = None
        self.table_grad_hook = None        # distributed.overlap_table_allreduce: called when the table gradient is parked
        self.tables._nsb_hash_ensemble = weakref.ref(self)
        self._register_state_dict_hook(self._to_reference_keys)
        self._register_load_state_dict_pre_hook(self._from_reference_keys)

    # -- reference-compatible views / checkpoints
    @property
    def hash_encodings(self) -> List[_GridView]:
        return [_GridView(self, c) for c in range(self.n_grids)]

    @torch.no_grad()
    def load_tcnn_grids(self, grids) -> None:
        """grids: 8 flat tensors in tcnn layout (what `hash_encodings.{c}.params` holds upstream)."""
        self.tables.copy_(packing.tables_from_tcnn([g.to(self.tables.device) for g in grids]))

    def tcnn_grids(self, tensor: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        return packing.tables_to_tcnn((self.tables if tensor is None else tensor).detach())

    @staticmethod
    def _to_reference_keys(module, state_dict, prefix, local_metadata):
        t = state_dict.pop(prefix + "tables")
        for c, g in enumerate(packing.tables_to_tcnn(t)):
            state_dict[f"{prefix}hash_encodings.{c}.params"] = g
        return state_dict

    def _from_reference_keys(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        keys = [f"{prefix}hash_encodings.{c}.params" for c in range(self.n_grids)]
        if all(k in state_dict for k in keys):
            state_dict[prefix + "tables"] = packing.tables_from_tcnn([state_dict.pop(k) for k in keys])

    # -- native fp16 table cache
    def native_tables(self) -> torch.Tensor:
        v = (self.tables._version, self.tables.data_ptr())
        if self._native is None or v != self._native_version:
            with torch.no_grad():
                self._native = self.tables.detach().half()
            self._native_version = v
        return self._native

    def shadow_buffer(self) -> torch.Tensor:
        if self._shadow is None or self._shadow.device != self.tables.device:
            self._shadow = torch.empty(self.tables.shape, dtype=torch.float16, device=self.tables.device)
        return self._shadow

    def materialize_pending(self, scale: float = 1.0) -> None:
        """Turn a parked rank-1 table gradient into a dense `.grad` (+=): gradient accumulation, dense all-reduce."""
        pend = self.pending_table_grad
        if pend is None:
            return
        g = ops.rank1_expand(pend, self.tables.shape[0], grad_scale=scale * float(pend.get("scale", 1.0)), out=self.tables.grad)
        if self.tables.grad is None:
            self.tables.grad = g
        self.pending_table_grad = None

    def set_native_tables(self, shadow: torch.Tensor) -> None:
        """The fused optimiser writes the fp16 copy itself; mark it current for the present value of `tables`."""
        self._native = shadow
        self._native_version = (self.tables._version, self.tables.data_ptr())

    def forward(self, in_tensor: torch.Tensor, conditioning_code: torch.Tensor, windows_param: Optional[float] = None,
                window_hash_encodings: Optional[float] = None) -> torch.Tensor:
        if windows_param is not None:
            raise NotImplementedError("per-level windowing (hash_ensemble.py:141-149, marked unused upstream)")
        assert conditioning_code.shape[-1] == self.n_hash_encodings, \
            "If blend mixing type is chosen, conditioning code needs to have as many dimensions as there are " \
            "hashtables in the encoding"
        if _needs_grad(in_tensor, conditioning_code, self.tables):
            return _HashEnsembleFunction.apply(self, in_tensor, conditioning_code, self.tables, window_hash_encodings)
        return ops.hash_blend_forward(self._blend_params(), in_tensor, conditioning_code, window_hash=window_hash_encodings,
                                      out_half=True, **self._blend_opts())

    def _blend_params(self) -> ops.NativeParams:
        return ops.NativeParams(self.native_tables(), None, None, None, None, torch.tensor([[0., 0, 0], [1, 1, 1]]),
                                self.levels, 1)

    def _blend_opts(self) -> dict:
        return dict(disable_initial=self.disable_initial_hash_ensemble, soft_transition=self.use_soft_transition)

    def get_out_dim(self) -> int:
        return self.n_output_dims

    def get_param_groups(self) -> Dict[str, List[nn.Parameter]]:
        return {"fields": [self.tables]}


@dataclass
class SE3DeformationFieldConfig:
    """deformation_field.py:15-21 (n_freq_pos is a plain class attribute upstream as well)."""
    n_freq_pos = 7
    warp_code_dim: int = 8
    mlp_num_layers: int = 6
    mlp_layer_width: int = 128
    skip_connections: Tuple[int] = (4,)


class _MLP(nn.Module):
    """Parameter container with nerfstudio MLP's module names (`layers.{i}.weight/bias`)."""

    def __init__(self, dims: List[Tuple[int, int]]):
        super().__init__()
        self.layers = nn.ModuleList([nn.Linear(i, o) for (o, i) in dims])


class SE3WarpingField(nn.Module):
    """deformation_field.py:32-75: parameters only (mlp_stem / mlp_r / mlp_v); evaluated inside the fused kernel."""

    def __init__(self, config: SE3DeformationFieldConfig):
        super().__init__()
        assert config.n_freq_pos == 7 and config.warp_code_dim == 128 and config.mlp_num_layers == 6 and \
            config.mlp_layer_width == 128 and tuple(config.skip_connections) == (4,), \
            "the CUDA kernels are specialised for the reference deformation field (7 freqs, 128-d code, 6x128, skip 4)"
        in_dim = 3 * 7 * 2 + 3 + config.warp_code_dim
        w = config.mlp_layer_width
        self.mlp_stem = _MLP([(w, in_dim), (w, w), (w, w), (w, w), (w, w + in_dim), (w, w)])
        self.mlp_r = _MLP([(3, w)])
        self.mlp_v = _MLP([(3, w)])
        nn.init.uniform_(self.mlp_r.layers[-1].weight, a=-1e-5, b=1e-5)
        nn.init.uniform_(self.mlp_v.layers[-1].weight, a=-1e-5, b=1e-5)
        nn.init.zeros_(self.mlp_r.layers[-1].bias)
        nn.init.zeros_(self.mlp_v.layers[-1].bias)

    def deform_dict(self):
        return dict(stem_w=[l.weight for l in self.mlp_stem.layers], stem_b=[l.bias for l in self.mlp_stem.layers],
                    r_w=self.mlp_r.layers[0].weight, r_b=self.mlp_r.layers[0].bias,
                    v_w=self.mlp_v.layers[0].weight, v_b=self.mlp_v.layers[0].bias)


class _DeformationFunction(torch.autograd.Function):
    """SE3DeformationField.compute_offsets with gradients for every se3_field parameter and the per-sample warp codes:
    nsb_field_forward (deformation only, saving the stem activations) / nsb_deform_backward."""

    @staticmethod
    def forward(ctx, field, positions, warp_code, window, *params):
        P = field._native_params()
        out = ops.field_forward(P, window_hash=None, window_deform=window, use_deformation=True, positions=positions,
                                sample_warp_codes=warp_code, want=("offsets", "deform_acts"))
        ctx.field, ctx.P, ctx.window = field, P, window
        ctx.saved = {"deform_acts": out["deform_acts"], "deform_enc": out["deform_enc"]}
        ctx.save_for_backward(positions, warp_code)
        return out["offsets"]

    @staticmethod
    @once_differentiable
    def backward(ctx, g_offsets):
        positions, warp_code = ctx.saved_tensors
        aabb = ctx.field.aabb.detach()
        d_xs = g_offsets.float() * (aabb[1] - aabb[0]).to(g_offsets.device)   # the offset enters the hash input as offset / size
        g = ops.deform_backward(ctx.P, ctx.saved, d_xs, window_deform=ctx.window, positions=positions,
                                sample_warp_codes=warp_code, loss_scale=float(ctx.field.mlp_loss_scale))
        grads = []
        for l in range(6):
            grads += [g["d_stem_w"][l], g["d_stem_b"][l]]
        grads += [g["d_r_w"], g["d_r_b"], g["d_v_w"], g["d_v_b"]]
        return (None, None, g["d_sample_warp_codes"], None) + tuple(grads)


class SE3DeformationField(nn.Module):
    """deformation_field.py:119-166."""

    def __init__(self, aabb: torch.Tensor, deformation_field_config: SE3DeformationFieldConfig,
                 max_n_samples_per_batch: int = -1):
        super().__init__()
        self.aabb = nn.Parameter(aabb, requires_grad=False)
        self.se3_field = SE3WarpingField(deformation_field_config)
        self.max_n_samples_per_batch = max_n_samples_per_batch   # kept for config compatibility; no chunking needed
        self.mlp_loss_scale = 128.0      # the backward's fp16 MLP deltas are scaled by this and the gradients divided back
        self._native = None
        self._native_version = None

    def _native_params(self) -> ops.NativeParams:
        v = tuple((p._version, p.data_ptr()) for p in self.parameters())
        if self._native is None or v != self._native_version:
            with torch.no_grad():
                self._native = ops.NativeParams.build(tables=None, time_emb=None, aabb=self.aabb.detach(),
                                                      levels=packing.level_table(), deform=self.se3_field.deform_dict(),
                                                      time_emb_deform=torch.zeros(1, 128), device=self.aabb.device)
            self._native_version = v
        return self._native

    def forward(self, ray_samples, warp_code: Optional[torch.Tensor] = None, windows_param: Optional[float] = None):
        assert ray_samples.frustums.offsets is None or (
            ray_samples.frustums.offsets == 0).all(), "ray samples have already been warped"
        positions = ray_samples.frustums.get_positions()
        ray_samples.frustums.set_offsets(self.compute_offsets(positions, warp_code, windows_param))
        return ray_samples

    def compute_offsets(self, positions: torch.Tensor, warp_code: Optional[torch.Tensor] = None,
                        windows_param: Optional[float] = None) -> torch.Tensor:
        """Offsets p' - p in NORMALISED aabb units (deformation_field.py:148-166)."""
        if warp_code is None:
            raise TypeError("warp_code is required (the reference would fail on `None - tensor`, deformation_field.py:162)")
        params = self._grad_params()
        if _needs_grad(positions, warp_code, *params):
            if positions.requires_grad:
                raise NotImplementedError(
                    "SE3DeformationField.compute_offsets: gradients w.r.t. the input positions (through the positional "
                    "encoding) are not implemented; detach the positions.  Parameters and warp codes get gradients.")
            return _DeformationFunction.apply(self, positions, warp_code, windows_param, *params)
        out = ops.field_forward(self._native_params(), window_hash=None, window_deform=windows_param, use_deformation=True,
                                positions=positions, sample_warp_codes=warp_code, want=("offsets",))
        return out["offsets"]

    def _grad_params(self) -> List[nn.Parameter]:
        """Parameters in the order _DeformationFunction returns their gradients."""
        f = self.se3_field
        ps = []
        for layer in f.mlp_stem.layers:
            ps += [layer.weight, layer.bias]
        return ps + [f.mlp_r.layers[0].weight, f.mlp_r.layers[0].bias, f.mlp_v.layers[0].weight, f.mlp_v.layers[0].bias]
