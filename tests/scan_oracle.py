"""Float64 references of the per-ray scan kernels on packed rays, each output with a rounding-error scale M:
compositing (render_weight_from_density + the white-background RGB, accumulation and clipped expected-depth renderers)
and its backward, the six training losses of models/base.py and their backward (as documented at the top of
csrc/nsb_losses.cu), and render_visibility_from_density.

Rays are evaluated in groups of equal sample count as [rays, count] tensors, so every prefix and suffix sum is a
cumulative sum along one ray, and a sum over no terms or over exact zeros is exactly 0.  (A cumulative sum over the whole
batch minus the segment start would leave ~1e-16 of the batch total there.)

Error scales.  M is the output's expression with every addend replaced by its absolute value and every transmittance
T_i = exp(-excl_i) replaced by T_i (1 + incl_i), incl_i = excl_i + sd_i: the kernels take excl_i as incl_i - sd_i from
an inclusive scan, so the rounding of the exponent scales with the inclusive sum, and exp turns that absolute error into
a relative one.  T_i exp(-sd_i) = exp(-incl_i) gets the same factor.  alpha = 1 - exp(-sd) becomes 1 + exp(-sd): its
float32 error is absolute, not relative (nerfacc's float32 arithmetic has the same rounding); it is 0 where sd = 0,
since alpha is then exactly 0 in float32 as well.  A quotient N / acc gets the first-order bound
(N_abs + |N / acc| acc_abs) / acc.  A later sample enters a sample's M only through a term that depends on that
sample, so M = 0 exactly where the float32 result has to be exactly 0.  A kernel output x then satisfies
|x - x64| <= error_constant(n) * U32 * M + floor.
"""
import math
from typing import Optional

import torch

U32 = 2.0 ** -24                                  # unit roundoff of float32
FLT_MIN = float(torch.finfo(torch.float32).tiny)
F64 = torch.float64


def error_constant(counts: torch.Tensor) -> torch.Tensor:
    """c(n), in units of U32, for a ray of n samples: a first-order count of the float32 roundings between the inputs
    and an output, each contributing at most U32 times the output's error scale M.
      - A warp scan (Hillis-Steele inclusive scan, or butterfly sum) passes every addend through 5 additions.
      - The carry between 32-sample chunks adds one addition per chunk: ceil(n / 32).
      - excl = carry + (incl - sd), and a suffix = carry + in-chunk suffix: 2 more.
      So one scan along the ray is at most 7 + ceil(n / 32) roundings deep.  Every output chains at most two such scans
      (transmittance, then the per-ray sum or the suffix of the per-sample terms; the near loss: the inclusive scan of
      w, then the suffix of the residuals): 2 (7 + ceil(n / 32)).
      - 24 for the fixed per-sample operations: sd = sigma dt; two expf (2 ulp each); 1 - e; T a; the seven additions
        and three products of G = dL/dw; G T e; the subtraction of the suffix and the product with dt.
    Nothing here is fitted to measured errors."""
    chunks = torch.div(counts.to(torch.int64) + 31, 32, rounding_mode="floor")
    return (2 * (7 + chunks) + 24).to(F64)


def _f64(x):
    return None if x is None else x.detach().to("cpu", F64)


def _groups(packed_info: torch.Tensor):
    """(ray ids [k], sample indices [k, n]) for each distinct non-zero sample count n."""
    info = packed_info.detach().to("cpu", torch.int64)
    start, cnt = info[:, 0], info[:, 1]
    for n in torch.unique(cnt).tolist():
        if n > 0:
            rays = torch.nonzero(cnt == n).flatten()
            yield rays, start[rays][:, None] + torch.arange(n)


def _excl_prefix(x):
    """sum_{j < i} along dim 1."""
    return torch.cat([torch.zeros_like(x[:, :1]), torch.cumsum(x, 1)[:, :-1]], 1)


def _excl_suffix(x):
    """sum_{j > i} along dim 1."""
    return _excl_prefix(x.flip(1)).flip(1)


def _incl_suffix(x):
    """sum_{j >= i} along dim 1."""
    return torch.cumsum(x.flip(1), 1).flip(1)


def _ray_terms(ts, te, sigma):
    """Per-sample quantities of [k, n] rays: the weights and their error scales."""
    dt = te - ts
    sd = sigma * dt
    incl = torch.cumsum(sd, 1)
    excl = torch.cat([torch.zeros_like(sd[:, :1]), incl[:, :-1]], 1)
    T, e = torch.exp(-excl), torch.exp(-sd)
    alpha = 1.0 - e            # not -expm1(-sd): torch's expm1 backward, 1 + expm1(x), rounds exp(-40) to 0
    w = T * alpha
    with torch.no_grad():
        grow = 1.0 + incl
        w_scale = T * grow * (1.0 + e) * (sd != 0)             # error scale of w = T a
        te_scale = T * e * grow                                # error scale of T e = exp(-incl)
    return dict(dt=dt, mid=(ts + te) / 2, sd=sd, incl=incl, T=T, e=e, alpha=alpha, w=w,
                w_scale=w_scale, te_scale=te_scale)


def _clip_range(t_starts, t_ends):
    mid = (_f64(t_starts) + _f64(t_ends)) / 2
    return (float(mid.min()), float(mid.max())) if mid.numel() else None


def composite(packed_info, t_starts, t_ends, sigma, rgb):
    """Training-mode composite: weights [S], rgb [R,3] (white background), accumulation [R], depth [R] (expected depth
    clipped to the batch's range of sample midpoints), and their error scales (*_scale)."""
    R = packed_info.shape[0]
    ts, te, sg, cc = map(_f64, (t_starts, t_ends, sigma, rgb))
    S = ts.shape[0]
    out = {"weights": torch.zeros(S, dtype=F64), "weights_scale": torch.zeros(S, dtype=F64),
           "rgb": torch.ones(R, 3, dtype=F64), "rgb_scale": torch.ones(R, 3, dtype=F64)}
    for k in ("accumulation", "accumulation_scale", "N", "N_scale"):
        out[k] = torch.zeros(R, dtype=F64)
    for rays, idx in _groups(packed_info):
        t = _ray_terms(ts[idx], te[idx], sg[idx])
        w, ws = t["w"], t["w_scale"]
        out["weights"][idx], out["weights_scale"][idx] = w, ws
        acc, acc_s = w.sum(1), ws.sum(1)
        out["accumulation"][rays], out["accumulation_scale"][rays] = acc, acc_s
        out["N"][rays], out["N_scale"][rays] = (w * t["mid"]).sum(1), (ws * t["mid"].abs()).sum(1)
        out["rgb"][rays] = (w[..., None] * cc[idx]).sum(1) + (1.0 - acc)[:, None]
        out["rgb_scale"][rays] = (ws[..., None] * cc[idx].abs()).sum(1) + (1.0 + acc_s)[:, None]
    acc, acc_s = out["accumulation"], out["accumulation_scale"]
    inv = 1.0 / (acc + 1e-10)
    draw = out["N"] * inv
    out["inv"], out["draw"] = inv, draw
    rng = _clip_range(t_starts, t_ends)
    out["clip"] = rng
    out["depth"] = draw.clamp(*rng) if rng else draw
    # the clip bounds are float32 midpoints in the kernel: + |lo| + |hi|
    out["depth_scale"] = ((out["N_scale"] + draw.abs() * (acc_s + 1e-10)) * inv + draw.abs() +
                          (abs(rng[0]) + abs(rng[1]) if rng else 0.0))
    return out


def composite_backward(packed_info, t_starts, t_ends, sigma, rgb, d_out_rgb, d_out_acc=None, d_out_depth=None,
                       d_weights=None):
    """Gradients of sum(d_out_rgb * rgb) + sum(d_out_acc * acc) + sum(d_out_depth * depth) + sum(d_weights * w) with
    respect to sigma [S] and the sample colours [S,3], by autograd in float64, and their error scales:
    returns (d_sigma, d_rgb, m_sigma, m_rgb).  The kernel's floor for d_sigma is FLT_MIN * dt."""
    R = packed_info.shape[0]
    ts, te, sg, cc = map(_f64, (t_starts, t_ends, sigma, rgb))
    S = ts.shape[0]
    g_rgb = _f64(d_out_rgb).reshape(R, 3)
    g_acc = torch.zeros(R, dtype=F64) if d_out_acc is None else _f64(d_out_acc).reshape(R)
    g_dep = torch.zeros(R, dtype=F64) if d_out_depth is None else _f64(d_out_depth).reshape(R)
    g_w = torch.zeros(S, dtype=F64) if d_weights is None else _f64(d_weights).reshape(S)
    fwd = composite(packed_info, t_starts, t_ends, sigma, rgb)
    rng = fwd["clip"]
    inv, draw = fwd["inv"], fwd["draw"]
    acc_s = fwd["accumulation_scale"] + 1e-10
    # torch.clip backward: the depth gradient passes only where lo <= depth <= hi
    g_dep_eff = g_dep * ((draw >= rng[0]) & (draw <= rng[1])) if rng else g_dep
    d_sigma, d_rgb = torch.zeros(S, dtype=F64), torch.zeros(S, 3, dtype=F64)
    m_sigma, m_rgb = torch.zeros(S, dtype=F64), torch.zeros(S, 3, dtype=F64)
    for rays, idx in _groups(packed_info):
        s = sg[idx].clone().requires_grad_(True)
        c = cc[idx].clone().requires_grad_(True)
        with torch.enable_grad():
            t = _ray_terms(ts[idx], te[idx], s)
            w = t["w"]
            acc = w.sum(1)
            depth = (w * t["mid"]).sum(1) / (acc + 1e-10)
            if rng:
                depth = torch.clamp(depth, rng[0], rng[1])
            out_rgb = (w[..., None] * c).sum(1) + (1.0 - acc)[:, None]
            L = ((out_rgb * g_rgb[rays]).sum() + (acc * g_acc[rays]).sum() + (depth * g_dep[rays]).sum() +
                 (w * g_w[idx]).sum())
            ds, dc = torch.autograd.grad(L, (s, c))
        d_sigma[idx], d_rgb[idx] = ds, dc
        # |G|: G = g_w + g_rgb . c - sum(g_rgb) + g_acc + g_dep (mid - draw) / acc, with the quotient's first-order bound
        mid, dr, iv = t["mid"], draw[rays][:, None], inv[rays][:, None]
        depth_term = g_dep_eff[rays].abs()[:, None] * iv * (
            mid.abs() + dr.abs() + (fwd["N_scale"][rays][:, None] + dr.abs() * acc_s[rays][:, None]) * iv +
            (mid - dr).abs() * acc_s[rays][:, None] * iv)
        G_abs = (g_w[idx].abs() + (g_rgb[rays][:, None, :] * cc[idx]).abs().sum(-1) + g_rgb[rays].sum(1).abs()[:, None] +
                 g_acc[rays].abs()[:, None] + depth_term)
        ws = t["w_scale"]
        m_sigma[idx] = t["dt"] * (G_abs * t["te_scale"] + _excl_suffix(G_abs * ws))
        m_rgb[idx] = g_rgb[rays].abs()[:, None, :] * ws[..., None]
    return d_sigma, d_rgb, m_sigma, m_rgb


def visibility(packed_info, t_starts, t_ends, sigma, early_stop_eps: float, alpha_thre: float):
    """render_visibility_from_density in float64: (visible [S] bool, ambiguous [S] bool).  A sample is ambiguous where
    float64 T or alpha is within the float32 error bound of its threshold, error_constant(n) * U32 * scale, the scale
    being T (1 + incl) for T and 1 + exp(-sd) for alpha."""
    ts, te, sg = map(_f64, (t_starts, t_ends, sigma))
    S = ts.shape[0]
    eps, thre = float(torch.tensor(early_stop_eps, dtype=torch.float32)), float(torch.tensor(alpha_thre, dtype=torch.float32))
    vis, amb = torch.zeros(S, dtype=torch.bool), torch.zeros(S, dtype=torch.bool)
    cnt = packed_info.detach().to("cpu", torch.int64)[:, 1]
    for rays, idx in _groups(packed_info):
        t = _ray_terms(ts[idx], te[idx], sg[idx])
        cu = error_constant(cnt[rays])[:, None] * U32
        v = t["T"] >= eps
        a = (t["T"] - eps).abs() < cu * t["T"] * (1.0 + t["incl"])
        if alpha_thre > 0:
            v = v & (t["alpha"] >= thre)
            a = a | ((t["alpha"] - thre).abs() < cu * (1.0 + t["e"]))
        vis[idx], amb[idx] = v, a
    return vis, amb


def _normal_cdf(x, scale):
    return 0.5 * (1.0 + torch.erf(x / (scale * math.sqrt(2.0))))


def losses(packed_info, t_starts, t_ends, weights, rgb, acc, depth, image, alpha: Optional[torch.Tensor],
           depth_target: Optional[torch.Tensor], cfg: dict, upstream):
    """The six losses (rgb, alpha, empty, near, depth, dist) and the gradients of sum_k upstream[k] * value[k] with
    respect to rgb [R,3], acc [R], depth [R] and the sample weights [S], in float64, with error scales.  cfg as in
    ops.losses_forward.  Returns a dict: values, d_rgb, d_acc, d_depth, d_weights and m_<each>."""
    R = packed_info.shape[0]
    cnt = packed_info.detach().to("cpu", torch.int64)[:, 1]
    ts, te = _f64(t_starts).reshape(-1), _f64(t_ends).reshape(-1)
    S = ts.shape[0]
    f32 = lambda v: float(torch.tensor(float(v), dtype=torch.float32))      # the kernels' float32 parameters
    lam = {k: f32(cfg.get(k) or 0.0) for k in ("lambda_alpha", "lambda_empty", "lambda_near", "lambda_depth", "lambda_dist")}
    eps = f32(cfg.get("eps_depth", 0.0))
    dist_max = int(cfg.get("dist_max_rays", 1 << 62))
    up = _f64(upstream).reshape(6)
    w = _f64(weights).reshape(S).requires_grad_(True)
    c = _f64(rgb).reshape(R, 3).requires_grad_(True)
    ac = _f64(acc).reshape(R).requires_grad_(True)
    dp = _f64(depth).reshape(R).requires_grad_(True)
    img = _f64(image).reshape(R, 3)
    al = None if alpha is None else _f64(alpha).reshape(R)
    tgt = None if depth_target is None else _f64(depth_target).reshape(R)
    ray_of = torch.repeat_interleave(torch.arange(R), cnt, output_size=S)
    mid, dt = (ts + te) / 2, te - ts
    one = lambda n: max(float(n), 1.0)

    # masks and counts (decided on the float32 inputs, away from their thresholds)
    masked = torch.ones(R, dtype=torch.bool)
    if cfg.get("use_masked_rgb", True) and al is not None:
        masked = al > f32(cfg.get("alpha_mask_threshold", 0.0))
    bg = (al < 1.0) if (al is not None and lam["lambda_alpha"] > 0) else torch.zeros(R, dtype=torch.bool)
    has_t = (tgt > 0) if tgt is not None else torch.zeros(R, dtype=torch.bool)
    t_s = tgt[ray_of] if tgt is not None else torch.zeros(S, dtype=F64)
    empty = has_t[ray_of] & (mid < t_s - eps) & (lam["lambda_empty"] > 0)
    near = has_t[ray_of] & (t_s - eps <= mid) & (mid <= t_s + eps) & (lam["lambda_near"] > 0)
    dm = has_t & (lam["lambda_depth"] > 0)
    sel_ray = (torch.arange(R) < dist_max) & (lam["lambda_dist"] > 0)
    has_sel = torch.nonzero(sel_ray & (cnt > 0)).flatten()
    n_sel = float(has_sel.max()) + 1.0 if has_sel.numel() else 1.0
    scale = (eps / 3.0) ** 2
    phi = _normal_cdf(mid - t_s, scale) if scale > 0 else torch.zeros(S, dtype=F64)
    # error scale of Phi(mid - tgt): its value, plus the rounding of mid and tgt (~U32 (|mid| + |tgt|)) through the
    # CDF's slope, which is up to 1 / (scale sqrt(2 pi)) ~ 29 at eps 0.35 (the variance is passed as the scale)
    phi_abs = 1.0 + (torch.exp(-0.5 * ((mid - t_s) / scale) ** 2) / (scale * math.sqrt(2.0 * math.pi)) * (mid.abs() + t_s.abs())
                     if scale > 0 else 0.0)
    n_mask, n_bg, n_vn, n_near, n_dm = (int(x.sum()) for x in (masked, bg, empty, near, dm))

    with torch.enable_grad():
        v = [None] * 6
        v[0] = ((img - c) ** 2)[masked].sum() / (3.0 * n_mask)
        v[1] = lam["lambda_alpha"] * (ac - al)[bg].abs().sum() / one(n_bg) if al is not None else ac.sum() * 0
        v[2] = lam["lambda_empty"] * (w[empty] ** 2).sum() / one(n_vn)
        v[4] = lam["lambda_depth"] * ((tgt - dp)[dm] ** 2).sum() / one(n_dm) if tgt is not None else dp.sum() * 0
        s_near = w.sum() * 0
        d1 = w.sum() * 0
        d2 = w.sum() * 0
        for rays, idx in _groups(packed_info):
            wg, mg = w[idx], mid[idx]
            A = torch.cumsum(wg, 1)
            s_near = s_near + (((A - phi[idx]) ** 2) * near[idx]).sum()
            sel = sel_ray[rays][:, None]
            d1 = d1 + (sel * dt[idx] * wg * wg).sum()
            d2 = d2 + (sel * wg * (mg * _excl_prefix(wg) - _excl_prefix(wg * mg))).sum()
        v[3] = lam["lambda_near"] * s_near / one(n_near)
        v[5] = lam["lambda_dist"] * ((1.0 / 3.0) * d1 + 2.0 * d2) / n_sel
        L = sum(up[k] * v[k] for k in range(6))
        gw, gc, ga, gd = torch.autograd.grad(L, (w, c, ac, dp), allow_unused=True)
    zero = lambda t, g: torch.zeros_like(t) if g is None else g
    out = {"values": torch.stack([x.detach() for x in v]), "d_weights": zero(w, gw), "d_rgb": zero(c, gc),
           "d_acc": zero(ac, ga), "d_depth": zero(dp, gd)}

    # error scales
    wa, ca, aca, dpa = w.detach().abs(), c.detach().abs(), ac.detach().abs(), dp.detach().abs()
    ce = abs(up[2]) * 2.0 * lam["lambda_empty"] / one(n_vn)
    cn = abs(up[3]) * 2.0 * lam["lambda_near"] / one(n_near)
    cd = abs(up[5]) * lam["lambda_dist"] / n_sel
    m_w = ce * wa * empty
    vs = torch.zeros(6, dtype=F64)
    vs[0] = ((img.abs() + ca) ** 2)[masked].sum() / (3.0 * max(n_mask, 1))
    if al is not None:
        vs[1] = lam["lambda_alpha"] * (aca + al.abs())[bg].sum() / one(n_bg)
    vs[2] = lam["lambda_empty"] * (wa[empty] ** 2).sum() / one(n_vn)
    if tgt is not None:
        vs[4] = lam["lambda_depth"] * ((tgt.abs() + dpa)[dm] ** 2).sum() / one(n_dm)
    for rays, idx in _groups(packed_info):
        wg, mg = wa[idx], mid[idx].abs()
        r_abs = (torch.cumsum(wg, 1) + phi_abs[idx]) * near[idx]
        m_w[idx] += cn * _incl_suffix(r_abs)
        vs[3] += lam["lambda_near"] * (r_abs ** 2).sum() / one(n_near)
        sel = sel_ray[rays][:, None]
        pre = mg * _excl_prefix(wg) + _excl_prefix(wg * mg)
        suf = _excl_suffix(wg * mg) + mg * _excl_suffix(wg)
        m_w[idx] += cd * sel * ((2.0 / 3.0) * dt[idx] * wg + 2.0 * (pre + suf))
        vs[5] += lam["lambda_dist"] * (sel * ((1.0 / 3.0) * dt[idx] * wg * wg + 2.0 * wg * pre)).sum() / n_sel
    out["m_weights"], out["m_values"] = m_w, vs
    out["m_rgb"] = (abs(up[0]) * 2.0 / (3.0 * max(n_mask, 1))) * (img.abs() + ca) * masked[:, None]
    out["m_acc"] = abs(up[1]) * lam["lambda_alpha"] / one(n_bg) * bg.to(F64)
    out["m_depth"] = (abs(up[4]) * 2.0 * lam["lambda_depth"] / one(n_dm)) * ((tgt.abs() if tgt is not None else 0.0) + dpa) * dm
    out["masks"] = {"masked": masked, "bg": bg, "empty": empty, "near": near, "depth": dm}
    return out
