"""CPU restatement of the reference's render hot path (functional, plain tensors).

TEST INFRASTRUCTURE (see oracle/__init__.py) -- never imported by the product.

Every function cites the reference file:line (relative to /root/reference/src/nersemble/)
it follows.  Third-party arithmetic comes from oracle/tp (tcnn / nerfacc / nerfstudio
restatements, [3P-mem], parity unpinned); the glue restated here is pinned by
tests/golden/*.npz, which oracle/gen_golden.py produced by running the REAL reference
modules (imported from /root/reference) on the same inputs.

Parameters are held in the kernels' native layout (FieldParams): one hash table
[entry][member(32)][feat(2)] instead of 8 tcnn grids of 8 features; `tables_from_tcnn` /
`tables_to_tcnn` convert (hash_ensemble.py:112 rearrange 'b c (l p f) -> b (l f) (c p)').

Precision modes (oracle.tp.tcnn_cpu.Precision.mode):
  "reference": fp16 roundings where the reference has them (tcnn half interpolation and
               outputs, fp16 window product / einsum output, autocast fp16 Linear outputs)
  "kernel":    roundings of the CUDA kernels (fp16-stored tables/weights, fp16 MLP inputs and
               hidden activations, fp32 everywhere else)
  "none":      fp16-stored tables/weights only
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from .tp import nerfacc_cpu as nerfacc
from .tp.tcnn_cpu import GridLevels, Precision, half_round, hashgrid_indices_weights, hashgrid_levels
from .tp.nerfstudio_cpu import trunc_exp


# ------------------------------------------------------------------------------------------
# parameters
# ------------------------------------------------------------------------------------------
@dataclass
class FieldParams:
    aabb: torch.Tensor                       # [2,3]
    tables: torch.Tensor                     # [N_entries, H, F] fp32 master (H=32 members, F=2)
    base_w: List[torch.Tensor]               # tcnn mlp_base weights [out,in]: [64,32],[16,64]
    head_w: List[torch.Tensor]               # tcnn mlp_head weights: [64,32],[64,64],[16,64]
    deform_w: List[torch.Tensor]             # nn.Linear weights of mlp_stem (6) [out,in]
    deform_b: List[torch.Tensor]
    r_w: torch.Tensor; r_b: torch.Tensor     # mlp_r Linear(128,3)
    v_w: torch.Tensor; v_b: torch.Tensor     # mlp_v Linear(128,3)
    time_emb: torch.Tensor                   # [T, H]   blend weights (nersemble_instant_ngp.py:116-118)
    time_emb_deform: torch.Tensor            # [T, Dw]  warp codes   (:120-125)
    levels: GridLevels = field(default_factory=hashgrid_levels)
    n_freq: int = 7
    skip_layer: int = 4
    geo_feat_dim: int = 15

    @property
    def n_timesteps(self):
        return self.time_emb.shape[0]

    def requires_grad_(self, flag=True):
        for t in self.all_tensors():
            t.requires_grad_(flag)
        return self

    def all_tensors(self):
        return ([self.tables] + self.base_w + self.head_w + self.deform_w + self.deform_b +
                [self.r_w, self.r_b, self.v_w, self.v_b, self.time_emb, self.time_emb_deform])


def tables_from_tcnn(grid_params: List[torch.Tensor], F: int = 2) -> torch.Tensor:
    """8 tcnn grids (flat [(entry)*8 + p*F + f]) -> native [entry, member=c*P+p, f].
    hash_ensemble.py:102-112: member h = c*P + p with P = 8/F, feature row d = l*F + f."""
    P = 8 // F
    per = [g.view(-1, P, F) for g in grid_params]          # [N, P, F] each
    return torch.stack(per, 1).reshape(per[0].shape[0], len(per) * P, F).contiguous()


def tables_to_tcnn(tables: torch.Tensor) -> List[torch.Tensor]:
    N, H, F = tables.shape
    P = 8 // F
    t = tables.view(N, H // P, P, F)
    return [t[:, c].reshape(-1).contiguous() for c in range(H // P)]


def random_params(seed: int = 19980801, n_timesteps: int = 4, log2_hashmap_size: int = 19,
                  table_scale: float = 1e-4, n_members: int = 32, deform_last_scale: float = 1e-5,
                  aabb=((-2.5, -1.8, -2.5), (2.2, 1.8, 2.0)), time_std_scale: float = 1.0) -> FieldParams:
    """Random-init parameters with the reference's init distributions (tcnn grid U(+-1e-4), tcnn MLP
    Xavier-uniform, nn.Linear default, last deformation layers U(+-1e-5)
    (deformation_field.py:72-75), time embeddings N(0, 0.01/sqrt(dim))
    (nersemble_instant_ngp.py:118,124)).  Seed = the reference's (train_nersemble.py:116)."""
    g = torch.Generator().manual_seed(seed)
    lv = hashgrid_levels(16, log2_hashmap_size, 16, 1.4472692012786865)
    N = lv.total_entries

    def U(shape, b):
        return (torch.rand(shape, generator=g) * 2 - 1) * b

    tables = U((N, n_members, 2), table_scale)

    def xavier(o, i):
        return U((o, i), math.sqrt(6.0 / (i + o)))

    base_w = [xavier(64, 32), xavier(16, 64)]
    head_w = [xavier(64, 32), xavier(64, 64), xavier(16, 64)]

    def lin(o, i):
        b = 1.0 / math.sqrt(i)
        return U((o, i), b), U((o,), b)

    dims = [(128, 173), (128, 128), (128, 128), (128, 128), (128, 301), (128, 128)]
    dw, db = [], []
    for (o, i) in dims:
        w, b = lin(o, i); dw.append(w); db.append(b)
    r_w = U((3, 128), deform_last_scale); v_w = U((3, 128), deform_last_scale)
    r_b = torch.zeros(3); v_b = torch.zeros(3)
    te = torch.randn((n_timesteps, n_members), generator=g) * (0.01 / math.sqrt(n_members)) * time_std_scale
    ted = torch.randn((n_timesteps, 128), generator=g) * (0.01 / math.sqrt(128)) * time_std_scale
    return FieldParams(torch.tensor(aabb, dtype=torch.float32), tables, base_w, head_w, dw, db,
                       r_w, r_b, v_w, v_b, te, ted, lv)


# ------------------------------------------------------------------------------------------
# schedulers / windows
# ------------------------------------------------------------------------------------------
def scheduler_value(step, init_value, final_value, begin_step, end_step):
    """engine/generic_scheduler.py:16-25."""
    if step > end_step:
        return final_value
    if step < begin_step:
        return init_value
    delta = min(max((step - begin_step) / (end_step - begin_step), 0), 1) * (final_value - init_value)
    return init_value + delta


def posenc_window(windows_param: float, min_bands: float, max_bands: float, dim: int) -> torch.Tensor:
    """field_components/hash_ensemble.py:12-28 == windowed_nerf_encoding.py:76-92."""
    bands = torch.linspace(min_bands, max_bands, dim)
    x = torch.clamp(windows_param - bands, 0, 1)
    return 0.5 * (1 - torch.cos(torch.pi * x))


# ------------------------------------------------------------------------------------------
# deformation field
# ------------------------------------------------------------------------------------------
def windowed_posenc(x: torch.Tensor, n_freq: int, windows_param: Optional[float]) -> torch.Tensor:
    """field_components/windowed_nerf_encoding.py:33-74 (include_input=True, covs=None).
    Output order: sin(x*f0..f6), sin(y*..), sin(z*..), cos(...)x21, then 2*pi*x (3)."""
    xt = 2 * torch.pi * x
    freqs = 2 ** torch.linspace(0.0, n_freq - 1, n_freq)
    scaled = (xt[..., None] * freqs).reshape(*xt.shape[:-1], -1)
    enc = torch.sin(torch.cat([scaled, scaled + torch.pi / 2.0], -1))
    if windows_param is not None:
        win = posenc_window(windows_param, 0.0, n_freq - 1, n_freq)[None, :].repeat(x.shape[-1], 1).reshape(-1).repeat(2)
        enc = win * enc
    return torch.cat([enc, xt], -1)


def _linear(x, w, b, mode):
    if mode == "reference" and Precision.autocast:
        # autocast fp16 Linear: operands and output fp16 (fp32 accumulate inside cuBLAS)
        return half_round(half_round(x) @ half_round(w).t() + half_round(b))
    if mode == "kernel":
        return half_round(x) @ half_round(w).t() + b
    return x @ w.t() + b


def deform_mlp(P: FieldParams, enc_in: torch.Tensor):
    """SE3WarpingField.get_transform MLP part (deformation_field.py:77-88) with nerfstudio MLP
    semantics: ReLU after every stem layer incl. the last (out_activation, :56); skip at layer 4
    concatenates [input, hidden] (:55)."""
    mode = Precision.mode
    x = enc_in
    for i, (w, b) in enumerate(zip(P.deform_w, P.deform_b)):
        if i == P.skip_layer:
            x = torch.cat([enc_in, x], -1)
        x = torch.relu(_linear(x, w, b, mode))
        if mode == "kernel":
            x = half_round(x)
    r = _linear(x, P.r_w, P.r_b, mode)
    v = _linear(x, P.v_w, P.v_b, mode)
    return r, v


def se3_apply(p: torch.Tensor, r: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """util/pytorch3d.py:107-191 (se3_exp_map with screw axis [v|r], eps=1e-4) followed by
    deformation_field.py:95-107: p' = R p + V v, NaN -> p.  Written with cross products:
    K p = r x p."""
    nrms = (r * r).sum(-1)
    theta = torch.clamp(nrms, 1e-4).sqrt()
    fac1 = theta.sin() / theta
    fac2 = (1.0 - theta.cos()) / (theta * theta)
    fac3 = (theta - theta.sin()) / (theta ** 3)
    rp = torch.cross(r, p, dim=-1); rrp = torch.cross(r, rp, dim=-1)
    rv = torch.cross(r, v, dim=-1); rrv = torch.cross(r, rv, dim=-1)
    Rp = p + fac1[:, None] * rp + fac2[:, None] * rrp
    Vv = v + fac2[:, None] * rv + fac3[:, None] * rrv
    out = Rp + Vv
    return torch.where(out.isnan(), p, out)


def compute_offsets(P: FieldParams, positions: torch.Tensor, warp_code: torch.Tensor,
                    window_deform: Optional[float]) -> torch.Tensor:
    """SE3DeformationField.compute_offsets (deformation_field.py:148-166): offsets in
    NORMALISED aabb units (later added to world positions -- reference quirk)."""
    pn = (positions - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    enc = windowed_posenc(pn, P.n_freq, window_deform)
    r, v = deform_mlp(P, torch.cat([enc, warp_code], -1))
    return se3_apply(pn, r.float(), v.float()) - pn


# ------------------------------------------------------------------------------------------
# hash ensemble + field MLPs
# ------------------------------------------------------------------------------------------
def blend_code(P: FieldParams, time_codes: torch.Tensor, window_hash: Optional[float],
               disable_initial: bool = True, soft_transition: bool = True):
    """hash_ensemble.py:119-139: returns (code [S,H], window [H] or None)."""
    H = time_codes.shape[-1]
    code = time_codes
    window = None
    if window_hash is not None:
        if window_hash == 1 and disable_initial:
            code = torch.ones_like(code)
        elif soft_transition and window_hash < 2:
            alpha = window_hash - 1
            code = alpha * code
            code = torch.cat([code[:, :1] + (1 - alpha), code[:, 1:]], -1)
        window = posenc_window(window_hash, 0, H - 1, H)
    return code, window


def hash_ensemble(P: FieldParams, x: torch.Tensor, time_codes: torch.Tensor,
                  window_hash: Optional[float]) -> torch.Tensor:
    """HashEnsemble.forward (hash_ensemble.py:93-158) on the native table layout.
    x [S,3] in [0,1); returns blended [S, L*F] (row d = l*F+f)."""
    mode = Precision.mode
    lv = P.levels
    S = x.shape[0]
    N, H, F = P.tables.shape
    idx, w = hashgrid_indices_weights(x.float(), lv)              # [S,L,8]
    L = lv.n_levels
    tab = half_round(P.tables)
    code, window = blend_code(P, time_codes, window_hash)
    if mode == "reference":
        # tcnn half interpolation per member -> fp16 embeddings [S, L*F, H]
        acc = torch.zeros(S, L, H, F)
        for c in range(8):
            vals = tab[idx[:, :, c].reshape(-1)].view(S, L, H, F)
            acc = half_round(half_round(w[:, :, c, None, None]) * vals + acc)
        emb = acc.permute(0, 1, 3, 2).reshape(S, L * F, H)       # [S, (l f), h]
        if window is not None:
            emb = half_round(half_round(window)[None, None, :] * emb)
        codeh = half_round(code)
        return half_round(torch.einsum("bdh,bh->bd", emb, codeh))
    cw = code if window is None else code * window[None, :]
    out = torch.zeros(S, L, F)
    for c in range(8):
        vals = tab[idx[:, :, c].reshape(-1)].view(S, L, H, F)
        inner = (vals * cw[:, None, :, None]).sum(2)                # [S,L,F]
        out = out + w[:, :, c, None] * inner
    return out.reshape(S, L * F)


def fused_mlp(x: torch.Tensor, weights: List[torch.Tensor], out_act: str) -> torch.Tensor:
    """tcnn FullyFusedMLP (bias-free, ReLU hidden); see oracle/tp/tcnn_cpu.Network."""
    mode = Precision.mode
    rnd = mode in ("reference", "kernel")
    h = half_round(x) if rnd else x
    for li, W in enumerate(weights):
        h = h @ half_round(W).t()
        if li < len(weights) - 1:
            h = torch.relu(h)
            if rnd:
                h = half_round(h)
    if mode == "reference":
        h = half_round(h)
    if out_act == "Sigmoid":
        h = torch.sigmoid(h)
        if mode == "reference":
            h = half_round(h)
    return h


def field_density(P: FieldParams, positions: torch.Tensor, time_codes: torch.Tensor,
                  window_hash: Optional[float]):
    """NeRSembleNeRFactoField.get_density (fields/nersemble_nerfacto_field.py:250-301)."""
    pn = (positions - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    selector = ((pn > 0.0) & (pn < 1.0)).all(-1)
    pn = pn * selector[..., None]
    feats = hash_ensemble(P, pn, time_codes, window_hash)
    h = fused_mlp(feats, P.base_w, "None")
    density = trunc_exp(h[:, :1].float()) * selector[..., None]
    return density, h[:, 1:1 + P.geo_feat_dim]


def field_rgb(P: FieldParams, directions: torch.Tensor, geo: torch.Tensor) -> torch.Tensor:
    """get_outputs (nersemble_nerfacto_field.py:303-383) with Identity direction encoding,
    no appearance embedding: h = cat[(d+1)/2, geo] -> pad to 32 with 1.0 -> mlp_head (sigmoid)."""
    d = (directions + 1.0) / 2.0
    h = torch.cat([d, geo.float()], -1)
    pad = 32 - h.shape[-1]
    h = torch.cat([h, torch.ones(h.shape[0], pad)], -1)
    return fused_mlp(h, P.head_w, "Sigmoid")[:, :3].float()


def timesteps_from_times(times: torch.Tensor, n_timesteps: int) -> torch.Tensor:
    """nersemble_instant_ngp.py:249,303: round(t*(T-1)) (torch.round = half-to-even)."""
    return (times * (n_timesteps - 1)).round().int().reshape(-1).long()


def field_density_fn(P: FieldParams, positions, times, window_hash, window_deform) -> torch.Tensor:
    """NeRSembleNGPModel.field_density_fn (nersemble_instant_ngp.py:235-266)."""
    ts = timesteps_from_times(times, P.n_timesteps)
    offsets = compute_offsets(P, positions, P.time_emb_deform[ts], window_deform)
    return field_density(P, positions + offsets, P.time_emb[ts], window_hash)[0]


# ------------------------------------------------------------------------------------------
# sampling
# ------------------------------------------------------------------------------------------
def fixed_samples(origins, directions, aabb, n_per_ray: int, step: float, near: float = 0.0):
    """BASELINE config-1/2 sampler: n_per_ray steps of `step` from the aabb entry
    (t0 = max(t_enter, near)); no occupancy grid.  Returns packed (t_starts, t_ends, ray_indices)."""
    import numpy as np
    R = origins.shape[0]
    o = origins.numpy().astype(np.float32); d = directions.numpy().astype(np.float32)
    a = aabb.reshape(-1).numpy().astype(np.float32)
    ts = np.zeros((R, n_per_ray), np.float32); te = np.zeros((R, n_per_ray), np.float32)
    for r in range(R):
        tmin, tmax, hit = nerfacc.ray_aabb_intersect_np(o[r], d[r], a)
        t = np.float32(max(tmin, np.float32(near))) if hit else np.float32(near)
        for k in range(n_per_ray):
            ts[r, k] = t
            t = np.float32(t + np.float32(step))
            te[r, k] = t
    ri = torch.arange(R).repeat_interleave(n_per_ray)
    return torch.from_numpy(ts.reshape(-1)), torch.from_numpy(te.reshape(-1)), ri


# ------------------------------------------------------------------------------------------
# full forward
# ------------------------------------------------------------------------------------------
def render(P: FieldParams, origins, directions, times, t_starts, t_ends, ray_indices,
           window_hash: Optional[float] = 32.0, window_deform: Optional[float] = 7.0,
           training: bool = False) -> Dict[str, torch.Tensor]:
    """NeRSembleNGPModel.get_outputs after the sampler (nersemble_instant_ngp.py:297-364)."""
    R = origins.shape[0]
    ri = ray_indices.long()
    ts = timesteps_from_times(times[ri], P.n_timesteps)                    # :303
    time_codes = P.time_emb[ts]                                             # :309
    warp_codes = P.time_emb_deform[ts]                                      # :315
    mid = (t_starts + t_ends)[:, None] / 2
    positions = origins[ri] + directions[ri] * mid                          # Frustums.get_positions
    offsets = compute_offsets(P, positions, warp_codes, window_deform)      # :320
    density, geo = field_density(P, positions + offsets, time_codes, window_hash)   # :322
    rgb = field_rgb(P, directions[ri], geo)
    packed_info = nerfacc.pack_info(ri, R)                                  # :325
    weights = nerfacc.render_weight_from_density(t_starts, t_ends, density[:, 0], packed_info)[0]  # :326-331
    # renderers (:334-343)
    rgb_in = rgb if training else torch.nan_to_num(rgb)
    comp = nerfacc.accumulate_along_rays(weights, rgb_in, ri, R)
    acc = nerfacc.accumulate_along_rays(weights, None, ri, R)
    comp = comp + (1.0 - acc)                                               # white background
    if not training:
        comp = comp.clamp(0.0, 1.0)
    steps = mid
    depth = nerfacc.accumulate_along_rays(weights, steps, ri, R) / (acc + 1e-10)
    if steps.numel():
        depth = torch.clip(depth, steps.min(), steps.max())
    deformation = nerfacc.accumulate_along_rays(weights, offsets, ri, R)   # deformation renderer :22-25
    return {"rgb": comp, "accumulation": acc, "depth": depth, "deformation": deformation,
            "num_samples_per_ray": packed_info[:, 1], "weights": weights[:, None], "offsets": offsets,
            "density": density, "rgb_samples": rgb, "positions": positions}


# ------------------------------------------------------------------------------------------
# occupancy sampler (NeRSembleVolumetricSampler.forward + OccGridEstimator.sampling)
# ------------------------------------------------------------------------------------------
def sample_occupancy(P: FieldParams, origins, directions, times, binaries, occs_mean: float,
                     render_step_size: float, near_plane: float, far_plane: float,
                     alpha_thre: float, early_stop_eps: float, cone_angle: float = 0.0,
                     training: bool = False, jitter: Optional[torch.Tensor] = None,
                     window_hash=None, window_deform=None, frustum_grid: Optional[torch.Tensor] = None):
    """model_components/nersemble_volumetric_sampler.py:44-135 on top of nerfacc sampling():
    frustum-cull mask AND (:90-93); stratified jitter only in training (:104); the visibility
    pre-pass (sigma_fn = field_density_fn at sample midpoints) only in training
    (VolumetricSampler.get_sigma_fn) with alpha_thre = min(alpha_thre, occs.mean());
    zero-sample guard (:110-115).  `jitter` [R] in [0,1) replaces torch.rand_like."""
    R = origins.shape[0]
    if frustum_grid is not None:
        binaries = binaries & frustum_grid[None]
    near = torch.full((R,), float(near_plane))
    far = torch.full((R,), float(far_plane))
    if training:
        near = near + jitter * render_step_size
    aabbs = P.aabb.reshape(1, 6)
    ts, te, ri = nerfacc.traverse_grids(origins, directions, binaries, aabbs, near, far, render_step_size, cone_angle)
    if training and (alpha_thre > 0.0 or early_stop_eps > 0.0):
        thre = min(alpha_thre, occs_mean)
        if ts.numel():
            pos = origins[ri] + directions[ri] * (ts + te)[:, None] / 2.0
            sig = field_density_fn(P, pos, times[ri], window_hash, window_deform).squeeze(-1)
        else:
            sig = torch.empty((0,))
        info = nerfacc.pack_info(ri, R)
        mask = nerfacc.render_visibility_from_density(ts, te, sig, packed_info=info,
                                                      early_stop_eps=early_stop_eps, alpha_thre=thre)
        ts, te, ri = ts[mask], te[mask], ri[mask]
    if ts.numel() == 0:
        ri = torch.zeros((1,), dtype=torch.long); ts = torch.ones((1,)); te = torch.ones((1,))
    return ts, te, ri


# ------------------------------------------------------------------------------------------
# losses (models/base.py:90-249 via nersemble_instant_ngp.py:366-407)
# ------------------------------------------------------------------------------------------
def loss_dict(out: Dict[str, torch.Tensor], t_starts, t_ends, ray_indices, batch: Dict[str, torch.Tensor],
              eps_depth: float, lam_alpha=1e-2, lam_near=1e-4, lam_empty=1e-2, lam_depth=1e-4, lam_dist=1e-4,
              alpha_mask_threshold: float = 0.0, dist_loss_max_rays: int = 5000,
              training: bool = True) -> Dict[str, torch.Tensor]:
    from .tp import flatten_eff_distloss
    losses = {}
    image = batch["image"]
    rgb = out["rgb"]; acc = out["accumulation"]; depth = out["depth"]; weights = out["weights"]
    ri = ray_indices.long()
    # masked rgb (base.py:90-118, use_masked_rgb_loss with alpha maps)
    alpha_per_ray = batch["alpha_map"].squeeze(1) / 255.0
    mask = alpha_per_ray > alpha_mask_threshold
    losses["rgb_loss"] = torch.nn.functional.mse_loss(image[mask], rgb[mask])
    # alpha (base.py:120-134)
    idx_bg = alpha_per_ray < 1
    if lam_alpha > 0 and idx_bg.any():
        losses["alpha_loss"] = (acc.squeeze(1)[idx_bg] - alpha_per_ray[idx_bg]).abs().mean() * lam_alpha
    # near / empty (base.py:136-204)
    if (lam_empty > 0 or lam_near > 0) and training:
        dt_ray = batch["depth_maps"]
        mid = (t_starts + t_ends) * 0.5
        tgt = dt_ray[ri]
        w = weights.squeeze(1)
        idx_very_near = (tgt > 0) & (mid < tgt - eps_depth)
        if lam_empty > 0 and idx_very_near.any():
            losses["empty_loss"] = lam_empty * (w[idx_very_near] ** 2).mean()
        if lam_near > 0:
            idx_near = (tgt > 0) & (tgt - eps_depth <= mid) & (mid <= tgt + eps_depth)
            normal = torch.distributions.Normal(0, (eps_depth / 3) ** 2)
            expected = normal.cdf(mid - tgt)
            if idx_near.any():
                info = nerfacc.pack_info(ri, acc.shape[0])
                accumulated = nerfacc.exclusive_sum(w, info) + w       # per-ray inclusive cumsum
                losses["near_loss"] = lam_near * ((accumulated[idx_near] - expected[idx_near]) ** 2).mean()
    # depth (base.py:206-222)
    if lam_depth > 0 and training:
        dt_ray = batch["depth_maps"]
        dm = dt_ray > 0
        if dm.any():
            losses["depth_loss"] = ((dt_ray[dm] - depth.squeeze()[dm]) ** 2).mean() * lam_depth
    # distortion (base.py:224-249)
    if lam_dist > 0:
        sel = ri < dist_loss_max_rays
        w = weights.squeeze(1)[sel]
        te_, ts_ = t_ends[sel], t_starts[sel]
        losses["dist_loss"] = lam_dist * flatten_eff_distloss(w, (te_ + ts_) * 0.5, te_ - ts_, ri[sel])
    return losses
