"""CPU restatement of the nerfacc 0.5.2 pieces the reference calls  [3P-mem].

TEST INFRASTRUCTURE (see oracle/__init__.py).  nerfacc==0.5.2+pt20cu117
(environment.yml:30-31) is not on disk; this restates its published behaviour:

  * OccGridEstimator (estimators/occ_grid.py): buffers, sampling(), _update(),
    update_every_n_steps()
  * traverse_grids / ray_aabb_intersect (csrc/grid.cu): DDA through the binary grid,
    fixed-step marching (dt = clamp(t*cone_angle, step, 1e10)), a sample is emitted
    while its midpoint lies before the current cell's exit and the cell is occupied
  * pack_info, exclusive_sum, render_transmittance_from_density,
    render_weight_from_density, render_visibility_from_density, accumulate_along_rays

Reference call sites: models/nersemble_instant_ngp.py:133-137,185-196,325-331;
model_components/nersemble_volumetric_sampler.py:95-108;
model_components/nersemble_deformation_renderer.py:22-25.

The marcher is a per-ray Python loop in numpy float32 scalars with the operation order
of the CUDA kernel (no fused multiply-add) so the CUDA marcher can be bit-exact to it.
PARITY UNPINNED for this layer (no nerfacc source / golden vectors available).

Upstream map (nerfacc v0.5.2, KAIR-BAIR/nerfacc):
  pack_info                          nerfacc/pack.py: pack_info (index_add_ counts, exclusive cumsum)
  exclusive_sum                      nerfacc/scan.py: exclusive_sum (packed segments)
  render_transmittance_from_density  nerfacc/volrend.py: render_transmittance_from_density (exp(-exclusive_sum(sigma*dt)))
  render_weight_from_density         nerfacc/volrend.py: render_weight_from_density (trans * alpha)
  render_visibility_from_density     nerfacc/volrend.py: render_visibility_from_density ((T >= eps) & (alpha >= thre))
  accumulate_along_rays              nerfacc/volrend.py: accumulate_along_rays (index_add_ over ray_indices)
  ray_aabb_intersect_np              nerfacc/cuda/csrc/grid.cu: device::ray_aabb_intersect / include/utils_grid.cuh
  _calc_dt                           nerfacc/cuda/csrc/include/utils_grid.cuh: calc_dt (clamp(t * cone_angle, dt_min, dt_max))
  traverse_ray / traverse_grids      nerfacc/cuda/csrc/grid.cu: device::traverse_grids_kernel (sorted aabb hits over
                                     levels, setup_traversal, the DDA with `continuous` skipping) behind
                                     nerfacc/grid.py: traverse_grids
  _enlarge_aabb                      nerfacc/grid.py: _enlarge_aabb
  OccGridEstimator                   nerfacc/estimators/occ_grid.py: OccGridEstimator.{__init__, sampling,
                                     update_every_n_steps, _get_all_cells, _sample_uniform_and_occupied_cells, _update}
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import numpy as np
import torch
from torch import nn

f32 = np.float32


# ----------------------------------------------------------------------------------------------
# packed-segment helpers
# ----------------------------------------------------------------------------------------------
def pack_info(ray_indices: torch.Tensor, n_rays: Optional[int] = None) -> torch.Tensor:
    if n_rays is None:
        n_rays = int(ray_indices.max()) + 1 if ray_indices.numel() else 0
    cnts = torch.zeros(n_rays, dtype=torch.long)
    cnts.index_add_(0, ray_indices.long(), torch.ones_like(ray_indices, dtype=torch.long))
    starts = cnts.cumsum(0) - cnts
    return torch.stack([starts, cnts], -1)


def _segment_ids(packed_info: torch.Tensor, n: int) -> torch.Tensor:
    cnts = packed_info[:, 1]
    return torch.repeat_interleave(torch.arange(len(cnts)), cnts, output_size=n)


def exclusive_sum(x: torch.Tensor, packed_info: torch.Tensor) -> torch.Tensor:
    """Per-segment exclusive prefix sum (differentiable)."""
    if x.numel() == 0:
        return x
    # float64 global cumsum: removes the cancellation error of (global prefix - segment start) in fp32
    xd = x.double()
    inc = torch.cumsum(xd, 0)
    seg = _segment_ids(packed_info, x.shape[0])
    starts = packed_info[:, 0]
    before = torch.cat([torch.zeros(1, dtype=torch.float64), inc])[starts]
    return (inc - xd - before[seg]).to(x.dtype)


def render_transmittance_from_density(t_starts, t_ends, sigmas, packed_info):
    sigmas_dt = sigmas * (t_ends - t_starts)
    alphas = 1.0 - torch.exp(-sigmas_dt)
    trans = torch.exp(-exclusive_sum(sigmas_dt, packed_info))
    return trans, alphas


def render_weight_from_density(t_starts, t_ends, sigmas, packed_info=None, ray_indices=None, n_rays=None,
                               prefix_trans=None):
    if packed_info is None:
        packed_info = pack_info(ray_indices, n_rays)
    trans, alphas = render_transmittance_from_density(t_starts, t_ends, sigmas, packed_info)
    weights = trans * alphas
    return weights, trans, alphas


def render_visibility_from_density(t_starts, t_ends, sigmas, packed_info=None, ray_indices=None, n_rays=None,
                                   early_stop_eps: float = 1e-4, alpha_thre: float = 0.0):
    if packed_info is None:
        packed_info = pack_info(ray_indices, n_rays)
    trans, alphas = render_transmittance_from_density(t_starts, t_ends, sigmas, packed_info)
    vis = trans >= early_stop_eps
    if alpha_thre > 0:
        vis = vis & (alphas >= alpha_thre)
    return vis


def accumulate_along_rays(weights, values=None, ray_indices=None, n_rays=None):
    if values is None:
        src = weights[..., None]
    else:
        src = weights[..., None] * values
    out = torch.zeros((n_rays, src.shape[-1]), dtype=src.dtype)
    out = out.index_add(0, ray_indices.long(), src)
    return out


# ----------------------------------------------------------------------------------------------
# ray marching (csrc/grid.cu)
# ----------------------------------------------------------------------------------------------
def ray_aabb_intersect_np(o: np.ndarray, d: np.ndarray, aabb: np.ndarray):
    """Slab test in float32, division by zero handled by IEEE inf.  Returns (tmin, tmax, hit)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = f32(1.0) / d
        t0 = (aabb[:3] - o) * inv
        t1 = (aabb[3:] - o) * inv
    tlo = np.minimum(t0, t1); thi = np.maximum(t0, t1)
    # NaN (0 * inf) slabs are ignored like fminf/fmaxf do
    tmin = f32(np.nanmax(tlo)) if not np.all(np.isnan(tlo)) else f32(-np.inf)
    tmax = f32(np.nanmin(thi)) if not np.all(np.isnan(thi)) else f32(np.inf)
    hit = bool(tmin <= tmax)
    return tmin, tmax, hit


def _calc_dt(t, cone_angle, dt_min, dt_max):
    return f32(min(max(f32(t * cone_angle), dt_min), dt_max))


def traverse_ray(o, d, binaries: np.ndarray, aabbs: np.ndarray, near, far, step, cone_angle):
    """One ray through `levels` nested grids.  o,d float32[3]; binaries bool[levels,X,Y,Z];
    aabbs float32[levels,6].  Returns (t_starts, t_ends) float32 lists."""
    levels = binaries.shape[0]
    res = np.array(binaries.shape[1:], np.int64)
    eps = f32(1e-6)
    step = f32(step); cone_angle = f32(cone_angle); near = f32(near); far = f32(far)
    # sorted intersections over levels
    tmins, tmaxs, hits = [], [], []
    for lv in range(levels):
        a, b, h = ray_aabb_intersect_np(o, d, aabbs[lv])
        if not h:
            a, b = f32(np.inf), f32(np.inf)     # miss_value
        tmins.append(a); tmaxs.append(b); hits.append(h)
    tvals = np.array(tmins + tmaxs, np.float32)
    order = np.argsort(tvals, kind="stable")
    t_sorted = tvals[order]

    ts, te = [], []
    t_last = near
    continuous = False
    with np.errstate(divide="ignore", invalid="ignore"):
        inv_d = f32(1.0) / d
    for i in range(2 * levels - 1):
        level = int(order[i] % levels)
        if not hits[level]:
            continue
        this_tmin = f32(max(t_sorted[i], near))
        this_tmax = f32(min(t_sorted[i + 1], far))
        if not (this_tmin < this_tmax):
            continue
        if not continuous:
            if step <= 0:
                t_last = this_tmin
            else:
                while True:
                    dt = _calc_dt(t_last, cone_angle, step, f32(1e10))
                    if f32(t_last + f32(dt * f32(0.5))) >= this_tmin:
                        break
                    t_last = f32(t_last + dt)
        amin = aabbs[level, :3]; amax = aabbs[level, 3:]
        resf = res.astype(np.float32)
        voxel = (amax - amin) / resf
        ray_start = o + d * f32(this_tmin + eps)
        ray_end = o + d * f32(this_tmax - eps)
        cur = np.clip((((ray_start - amin) / (amax - amin)) * resf).astype(np.int64), 0, res - 1)
        fin = np.clip((((ray_end - amin) / (amax - amin)) * resf).astype(np.int64), 0, res - 1)
        index_delta = (d > 0).astype(np.int64)
        start_index = cur + index_delta
        with np.errstate(invalid="ignore"):
            tmax_xyz = ((amin + (start_index.astype(np.float32) * voxel - ray_start)) * inv_d) + this_tmin
        tdist = np.where(d == 0, this_tmax, tmax_xyz).astype(np.float32)
        step_f = np.where(d == 0, f32(0), np.where(d > 0, f32(1), f32(-1))).astype(np.float32)
        step_i = step_f.astype(np.int64)
        with np.errstate(invalid="ignore"):
            delta = np.where(d == 0, this_tmax, voxel * inv_d * step_f).astype(np.float32)
        overflow = fin + step_i
        while True:
            t_trav = f32(min(min(tdist[0], min(tdist[1], tdist[2])), this_tmax))
            occupied = bool(binaries[level, cur[0], cur[1], cur[2]])
            if not occupied:
                if step <= 0:
                    t_last = t_trav
                else:
                    while True:
                        dt = _calc_dt(t_last, cone_angle, step, f32(1e10))
                        if f32(t_last + f32(dt * f32(0.5))) >= t_trav:
                            break
                        t_last = f32(t_last + dt)
                continuous = False
            else:
                while True:
                    if step <= 0:
                        t_next = t_trav
                    else:
                        dt = _calc_dt(t_last, cone_angle, step, f32(1e10))
                        if f32(t_last + f32(dt * f32(0.5))) >= t_trav:
                            break
                        t_next = f32(t_last + dt)
                    ts.append(t_last); te.append(t_next)
                    continuous = True
                    t_last = t_next
                    if t_next >= t_trav:
                        break
            # single_traversal
            if tdist[0] < tdist[1] and tdist[0] < tdist[2]:
                ax = 0
            elif tdist[1] < tdist[2]:
                ax = 1
            else:
                ax = 2
            cur[ax] += step_i[ax]
            tdist[ax] = f32(tdist[ax] + delta[ax])
            if cur[ax] == overflow[ax]:
                break
    return ts, te


def traverse_grids(rays_o: torch.Tensor, rays_d: torch.Tensor, binaries: torch.Tensor, aabbs: torch.Tensor,
                   near_planes: torch.Tensor, far_planes: torch.Tensor, step_size: float, cone_angle: float):
    o = rays_o.detach().cpu().numpy().astype(np.float32)
    d = rays_d.detach().cpu().numpy().astype(np.float32)
    b = binaries.detach().cpu().numpy().astype(bool)
    a = aabbs.detach().cpu().numpy().astype(np.float32)
    nearp = near_planes.detach().cpu().numpy().astype(np.float32)
    farp = far_planes.detach().cpu().numpy().astype(np.float32)
    all_ts, all_te, all_ri = [], [], []
    for r in range(o.shape[0]):
        ts, te = traverse_ray(o[r], d[r], b, a, nearp[r], farp[r], step_size, cone_angle)
        all_ts += ts; all_te += te; all_ri += [r] * len(ts)
    t_starts = torch.tensor(np.array(all_ts, np.float32)).reshape(-1)
    t_ends = torch.tensor(np.array(all_te, np.float32)).reshape(-1)
    ray_indices = torch.tensor(np.array(all_ri, np.int64)).reshape(-1)
    return t_starts, t_ends, ray_indices


def _enlarge_aabb(aabb: torch.Tensor, factor: float) -> torch.Tensor:
    center = (aabb[:3] + aabb[3:]) / 2
    extent = (aabb[3:] - aabb[:3]) / 2
    return torch.cat([center - extent * factor, center + extent * factor])


class OccGridEstimator(nn.Module):
    """estimators/occ_grid.py (0.5.2)."""

    DIM = 3

    def __init__(self, roi_aabb, resolution=128, levels: int = 1, **kwargs):
        super().__init__()
        if isinstance(resolution, int):
            resolution = [resolution] * 3
        resolution = torch.tensor(resolution, dtype=torch.int32)
        roi_aabb = torch.as_tensor(roi_aabb, dtype=torch.float32).flatten()
        aabbs = torch.stack([_enlarge_aabb(roi_aabb, 2 ** i) for i in range(levels)], 0)
        self.cells_per_lvl = int(resolution.prod().item())
        self.levels = levels
        self.register_buffer("resolution", resolution)
        self.register_buffer("aabbs", aabbs)
        self.register_buffer("occs", torch.zeros(self.levels * self.cells_per_lvl))
        self.register_buffer("binaries", torch.zeros([levels] + resolution.tolist(), dtype=torch.bool))
        gx, gy, gz = torch.meshgrid(*[torch.arange(int(r)) for r in resolution], indexing="ij")
        grid_coords = torch.stack([gx, gy, gz], -1).reshape(self.cells_per_lvl, 3)
        self.register_buffer("grid_coords", grid_coords, persistent=False)
        self.register_buffer("grid_indices", torch.arange(self.cells_per_lvl), persistent=False)

    @property
    def device(self):
        return self.occs.device

    @torch.no_grad()
    def sampling(self, rays_o, rays_d, sigma_fn: Optional[Callable] = None, alpha_fn=None,
                 near_plane: float = 0.0, far_plane: float = 1e10, t_min=None, t_max=None,
                 render_step_size: float = 1e-3, early_stop_eps: float = 1e-4, alpha_thre: float = 0.0,
                 stratified: bool = False, cone_angle: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        near_planes = torch.full_like(rays_o[..., 0], fill_value=near_plane)
        far_planes = torch.full_like(rays_o[..., 0], fill_value=far_plane)
        if t_min is not None:
            near_planes = torch.clamp(near_planes, min=t_min)
        if t_max is not None:
            far_planes = torch.clamp(far_planes, max=t_max)
        if stratified:
            near_planes += torch.rand_like(near_planes) * render_step_size
        t_starts, t_ends, ray_indices = traverse_grids(
            rays_o, rays_d, self.binaries, self.aabbs, near_planes, far_planes, render_step_size, cone_angle)
        packed_info = pack_info(ray_indices, rays_o.shape[0])
        if (alpha_thre > 0.0 or early_stop_eps > 0.0) and (sigma_fn is not None or alpha_fn is not None):
            alpha_thre = min(alpha_thre, self.occs.mean().item())
            if t_starts.shape[0] != 0:
                sigmas = sigma_fn(t_starts, t_ends, ray_indices)
            else:
                sigmas = torch.empty((0,))
            assert sigmas.shape == t_starts.shape
            masks = render_visibility_from_density(t_starts, t_ends, sigmas, packed_info=packed_info,
                                                   early_stop_eps=early_stop_eps, alpha_thre=alpha_thre)
            ray_indices, t_starts, t_ends = ray_indices[masks], t_starts[masks], t_ends[masks]
        return ray_indices, t_starts, t_ends

    @torch.no_grad()
    def update_every_n_steps(self, step: int, occ_eval_fn: Callable, occ_thre: float = 1e-2,
                             ema_decay: float = 0.95, warmup_steps: int = 256, n: int = 16) -> None:
        if not self.training:
            raise RuntimeError("You should only call this function only during training.")
        if step % n == 0 and self.training:
            self._update(step, occ_eval_fn, occ_thre, ema_decay, warmup_steps)

    @torch.no_grad()
    def _get_all_cells(self):
        return [self.grid_indices] * self.levels

    @torch.no_grad()
    def _sample_uniform_and_occupied_cells(self, n: int):
        lvl_indices = []
        for lvl in range(self.levels):
            uniform_indices = torch.randint(self.cells_per_lvl, (n,))
            occupied_indices = torch.nonzero(self.binaries[lvl].flatten())[:, 0]
            if n < len(occupied_indices):
                selector = torch.randint(len(occupied_indices), (n,))
                occupied_indices = occupied_indices[selector]
            lvl_indices.append(torch.cat([uniform_indices, occupied_indices], 0))
        return lvl_indices

    @torch.no_grad()
    def _update(self, step, occ_eval_fn, occ_thre=0.01, ema_decay=0.95, warmup_steps=256):
        if step < warmup_steps:
            indices_all = self._get_all_cells()
        else:
            indices_all = self._sample_uniform_and_occupied_cells(self.cells_per_lvl // 4)
        for lvl, indices in enumerate(indices_all):
            grid_coords = self.grid_coords[indices]
            x = (grid_coords + torch.rand_like(grid_coords, dtype=torch.float32)) / self.resolution
            x = self.aabbs[lvl, :3] + x * (self.aabbs[lvl, 3:] - self.aabbs[lvl, :3])
            occ = occ_eval_fn(x).squeeze(-1)
            cell_ids = lvl * self.cells_per_lvl + indices
            self.occs[cell_ids] = torch.maximum(self.occs[cell_ids] * ema_decay, occ.float())
        thre = torch.clamp(self.occs[self.occs >= 0].mean(), max=occ_thre)
        self.binaries = (self.occs > thre).view(self.binaries.shape)
