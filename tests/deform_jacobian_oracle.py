"""CPU oracle of the deformation's input Jacobian and of observation-space normals, on top of oracle.pipeline (plain torch,
differentiable as written): J = d offset / d p_n by autograd through compute_offsets, and the observation-space gradient of
h0 composed by the chain rule through the hash input x = s (p_n + D^-1 offset(p_n)), D = diag(box extent)."""
from typing import Optional

import torch

from normals_oracle import h0
from oracle import pipeline as pl


def _extent(P):
    return P.aabb[1] - P.aabb[0]


def offsets_of_normalised(P, pn: torch.Tensor, warp_code: torch.Tensor, window_deform) -> torch.Tensor:
    """Normalised offsets as a function of the normalised position (compute_offsets takes world positions)."""
    return pl.compute_offsets(P, P.aabb[0] + pn * _extent(P), warp_code, window_deform)


def offsets_vjp(P, positions: torch.Tensor, warp_code: torch.Tensor, window_deform, u: torch.Tensor, chunk: int = 8192):
    """J^T u [n,3] with respect to the NORMALISED position, for world `positions` and a cotangent u of the offsets."""
    pn_all = ((positions.float() - P.aabb[0]) / _extent(P)).detach()
    out = []
    for i in range(0, pn_all.shape[0], chunk):
        pn = pn_all[i:i + chunk].clone().requires_grad_(True)
        with torch.enable_grad():
            off = offsets_of_normalised(P, pn, warp_code[i:i + chunk], window_deform)
            g, = torch.autograd.grad((off * u[i:i + chunk]).sum(), pn)
        out.append(g)
    return torch.cat(out) if out else torch.zeros((0, 3))


def jacobian_norm(P, positions, warp_code, window_deform) -> torch.Tensor:
    """Frobenius norm of J per sample (three pullbacks of the unit vectors)."""
    cols = [offsets_vjp(P, positions, warp_code, window_deform, torch.eye(3)[k].expand(positions.shape[0], 3)) for k in range(3)]
    return torch.stack(cols, -1).norm(dim=(-2, -1))


def observation_normals(P, positions, warp_code, time_codes, window_hash, window_deform, world_space: bool = False,
                        blend_fp16: bool = False, offsets: Optional[torch.Tensor] = None, chunk: int = 4096):
    """(normals [n,3], gradient [n,3], selector [n]): d h0 / d p_n = s (g + J^T D^-1 g) with g = d h0 / d x at the warped
    position, divided by the extent once more when world_space; normals = -gradient / max(|gradient|, 1e-12), the zero
    vector where the warped position is outside the box (s = 0).  offsets: evaluate g at positions + offsets (the
    kernels' own warp) instead of the oracle's; J always comes from the oracle's deformation."""
    ext = _extent(P)
    grads, sels = [], []
    for i in range(0, positions.shape[0], chunk):
        pos, wc, tc = positions[i:i + chunk].float(), warp_code[i:i + chunk], time_codes[i:i + chunk]
        with torch.no_grad():
            off = pl.compute_offsets(P, pos, wc, window_deform) if offsets is None else offsets[i:i + chunk].float()
            xw = (pos + off - P.aabb[0]) / ext
            sel = ((xw > 0.0) & (xw < 1.0)).all(-1)
        x = (xw * sel[:, None]).detach().requires_grad_(True)
        with torch.enable_grad():
            g, = torch.autograd.grad(h0(P, x, tc, window_hash, blend_fp16).sum(), x)
        v = sel[:, None] * (g + offsets_vjp(P, pos, wc, window_deform, g / ext))
        grads.append(v / ext if world_space else v)
        sels.append(sel)
    g = torch.cat(grads)
    return -g / g.norm(dim=-1, keepdim=True).clamp_min(1e-12), g, torch.cat(sels)
