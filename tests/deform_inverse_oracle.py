"""CPU oracle of the deformation's forward-mode Jacobian and of its inverse, on top of oracle.pipeline: J by torch.func.jacfwd
(and by the three pullbacks of deform_jacobian_oracle), and a float64 damped-Newton solve of
F(p_n) = p_n + D^-1 offset(p_n) - c_n = 0 with the kernel's rule."""
import dataclasses

import torch

from deform_jacobian_oracle import offsets_vjp
from oracle import pipeline as pl


def jacobian_by_pullbacks(P, positions, warp_code, window_deform) -> torch.Tensor:
    """[n,3,3] with J[:, i, :] = J^T e_i (autograd through oracle.pipeline)."""
    n = positions.shape[0]
    return torch.stack([offsets_vjp(P, positions, warp_code, window_deform, torch.eye(3)[i].expand(n, 3)) for i in range(3)], 1)


def offsets_any_dtype(P, pn: torch.Tensor, warp_code: torch.Tensor, window_deform) -> torch.Tensor:
    """compute_offsets of normalised positions, composed from oracle.pipeline's pieces without its float32 casts, so
    that float64 parameters (as_float64) give a float64 warp."""
    enc = pl.windowed_posenc(pn, P.n_freq, window_deform)
    r, v = pl.deform_mlp(P, torch.cat([enc, warp_code.to(enc.dtype)], -1))
    return pl.se3_apply(pn, r, v) - pn


def jacobian_jacfwd(P, pn: torch.Tensor, warp_code: torch.Tensor, window_deform) -> torch.Tensor:
    """[n,3,3] J[i][k] = d offset_i / d pn_k by forward-mode AD (torch.func.jacfwd, vmapped over the points)."""
    from torch.func import jacfwd, vmap

    def one(p, wc):
        return offsets_any_dtype(P, p[None], wc[None], window_deform)[0]

    return vmap(jacfwd(one, argnums=0))(pn, warp_code)


def as_float64(P):
    """The deformation part of P in float64 (the hash tables are not needed by the warp)."""
    d = lambda t: t.detach().double()
    return dataclasses.replace(P, aabb=d(P.aabb), deform_w=[d(w) for w in P.deform_w], deform_b=[d(b) for b in P.deform_b],
                               r_w=d(P.r_w), r_b=d(P.r_b), v_w=d(P.v_w), v_b=d(P.v_b))


def newton_inverse(P64, targets: torch.Tensor, warp_code: torch.Tensor, window_deform, init=None, max_iter: int = 60,
                   tol: float = 1e-13):
    """float64 damped Newton with the kernel's rule: a trial with a smaller |F|inf than the best becomes the best and the
    next trial is best - (I + D^-1 J)^-1 F; any other trial is replaced by the midpoint with the best.  Needs
    Precision.mode = "none" (no fp16 rounding).  Returns (positions world [n,3], residual [n])."""
    ext = P64.aabb[1] - P64.aabb[0]
    cn = (targets.double() - P64.aabb[0]) / ext
    wc = warp_code.double()
    trial = cn.clone() if init is None else (init.double() - P64.aabb[0]) / ext
    best = trial.clone()
    rbest = torch.full((cn.shape[0],), float("inf"), dtype=torch.float64)
    eye = torch.eye(3, dtype=torch.float64)
    for _ in range(max_iter + 1):
        with torch.no_grad():
            off = offsets_any_dtype(P64, trial, wc, window_deform)
        F = trial + off / ext - cn
        r = F.abs().amax(-1)
        better = r < rbest
        best = torch.where(better[:, None], trial, best)
        rbest = torch.where(better, r, rbest)
        if (rbest < tol).all():
            break
        J = jacobian_jacfwd(P64, trial, wc, window_deform)
        step = torch.linalg.solve(eye + J / ext[:, None], F)
        trial = torch.where(better[:, None], best - step, 0.5 * (best + trial))
    return P64.aabb[0] + best * ext, rbest


def rigid_inverse(c_n: torch.Tensor, r, v) -> torch.Tensor:
    """The analytic inverse of the rigid warp x = R p + V v (unit box): R^-1 (c - V v), float64.  R^-1 = R^T except in the
    clamp branch (theta^2 < 1e-4), where the map's R is I + f1 K + f2 K^2 with theta clamped and not exactly orthogonal."""
    r = torch.as_tensor(r, dtype=torch.float64)
    v = torch.as_tensor(v, dtype=torch.float64)
    th = (r * r).sum().clamp_min(1e-4).sqrt()
    K = torch.tensor([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]], dtype=torch.float64)
    R = torch.eye(3, dtype=torch.float64) + (th.sin() / th) * K + ((1 - th.cos()) / th ** 2) * (K @ K)
    V = torch.eye(3, dtype=torch.float64) + ((1 - th.cos()) / th ** 2) * K + ((th - th.sin()) / th ** 3) * (K @ K)
    return torch.linalg.solve(R, (c_n.double() - V @ v).T).T


def rigid_params(r, v):
    """Unit-cube box, stem weights and biases zero (a5 = 0), head biases (r, v): the warp is x = R p_n + V v everywhere."""
    P = pl.random_params(n_timesteps=2, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
                         aabb=((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)))
    for w, b in zip(P.deform_w, P.deform_b):
        w.zero_(); b.zero_()
    P.r_b.copy_(torch.tensor(r)); P.v_b.copy_(torch.tensor(v))
    return P
