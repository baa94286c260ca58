"""CPU oracle of the surface normals (nerfstudio 0.3.1 Field.get_normals and NormalsRenderer(normalize=True)) on top of
oracle.pipeline: autograd of h0 (mlp_base output 0 before trunc_exp) with respect to the masked normalised position
x = selector * (p - aabb_min) / (aabb_max - aabb_min) (fields/nersemble_nerfacto_field.py:257-287).  The oracle's hash
grid is differentiable in x with d frac / dx = scale (oracle/tp/tcnn_cpu.py)."""
from typing import Optional

import torch

from oracle import pipeline as pl


def masked_position(P, positions: torch.Tensor, offsets: Optional[torch.Tensor] = None) -> torch.Tensor:
    p = positions if offsets is None else positions + offsets
    pn = (p - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    selector = ((pn > 0.0) & (pn < 1.0)).all(-1)
    return pn * selector[..., None]


def h0(P, x: torch.Tensor, time_codes: torch.Tensor, window_hash, blend_fp16: bool = False) -> torch.Tensor:
    """blend_fp16: the member weights (code x window) rounded to fp16 first, as the kernels' per-sample line gather
    rounds them (its MMA operand); the blended frame tables keep them in fp32, as the oracle does."""
    if blend_fp16:
        code, window = pl.blend_code(P, time_codes, window_hash)
        time_codes, window_hash = (code if window is None else code * window[None, :]).half().float(), None
    return pl.fused_mlp(pl.hash_ensemble(P, x, time_codes, window_hash), P.base_w, "None")[:, 0]


def field_normals(P, positions, time_codes, window_hash, offsets=None, world_space: bool = False, chunk: int = 4096,
                  blend_fp16: bool = False):
    """(normals [n,3], gradient d h0 / dx [n,3]) -- the gradient divided by the box extent when world_space."""
    x_all = masked_position(P, positions.float(), None if offsets is None else offsets.float()).detach()
    grads = []
    for i in range(0, x_all.shape[0], chunk):
        x = x_all[i:i + chunk].clone().requires_grad_(True)
        with torch.enable_grad():
            g, = torch.autograd.grad(h0(P, x, time_codes[i:i + chunk], window_hash, blend_fp16).sum(), x)
        grads.append(g)
    g = torch.cat(grads) if grads else torch.zeros((0, 3))
    if world_space:
        g = g / (P.aabb[1] - P.aabb[0])
    return -torch.nn.functional.normalize(g, dim=-1), g


def composite_normals(normals: torch.Tensor, weights: torch.Tensor, ray_indices: torch.Tensor, n_rays: int) -> torch.Tensor:
    """NormalsRenderer(normalize=True) on packed samples: safe_normalize(sum_i w_i n_i), v / (|v| + 1e-10)."""
    v = torch.zeros((n_rays, 3), dtype=normals.dtype).index_add_(0, ray_indices.long(), weights.reshape(-1, 1) * normals)
    return v / (v.norm(dim=-1, keepdim=True) + 1e-10)
