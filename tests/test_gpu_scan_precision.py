"""The per-ray scan kernels (compositing forward and backward, the fused losses' backward, the visibility filter)
against the float64 references of tests/scan_oracle.py, sample by sample, on one batch of long, opaque and
degenerate rays.  Every output x must satisfy |x - x64| <= c(n) * U32 * M + floor, with M the float64 error scale of
that output and c(n) the rounding count derived in scan_oracle.error_constant; where M = 0 (no later sample the
output depends on carries weight), x must be exactly 0."""
import pytest
import torch

import scan_oracle as so

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = 0.011
SHORT = [0, 1, 31, 32, 33, 63, 64, 65, 256]          # 256: the fixed-stride config-3 ray
PROFILES = ["zeros", "opaque_first", "shell", "shell_fp32", "excl_cross", "tiny", "huge", "random"]


def _profile(name, n, g):
    """sigma * dt of one ray."""
    u = lambda lo, hi: torch.rand(n, generator=g, dtype=torch.float64) * (hi - lo) + lo
    if name == "zeros" or n == 0:
        return torch.zeros(n, dtype=torch.float64)
    if name == "opaque_first":                        # every later float32 (and float64) weight is exactly 0
        sd = u(0, 2); sd[0] = 1000.0; return sd
    if name in ("shell", "shell_fp32"):               # density, an opaque shell in the middle, density behind it
        sd = u(0, 0.05)
        k = n // 2
        sd[k:k + 4] = 400.0 if name == "shell" else 40.0      # float64 T behind: 0, or ~1e-70 (float32: 0)
        sd[k + 4:] = u(0, 2)[k + 4:]
        return sd
    if name == "excl_cross":                          # excl runs through 88..104, where expf goes denormal, then 0
        sd = torch.full((n,), 30.0 / max(n - 1, 1), dtype=torch.float64); sd[0] = 80.0; return sd
    if name == "tiny":
        return u(0.5e-6, 1.5e-6)
    if name == "huge":
        return u(0.5e3, 1.5e3)
    sd = u(0, 0.5); sd[torch.rand(n, generator=g) < 0.2] = 0.0; return sd


@pytest.fixture(scope="module")
def batch():
    """4096 rays: the SHORT counts in turn, 64 rays of 1000 and 64 of 4097 samples, every count with every profile;
    the last ray is a zero-density guard with the batch's lowest and highest midpoints, so that no other ray's
    expected depth sits on a clip bound."""
    g = torch.Generator().manual_seed(20261016)
    R = 4096
    counts, prof = [], []
    for r in range(R - 1):
        if r % 64 == 5:
            counts.append(1000); prof.append(PROFILES[(r // 64) % len(PROFILES)])
        elif r % 64 == 37:
            counts.append(4097); prof.append(PROFILES[(r // 64) % len(PROFILES)])
        else:
            counts.append(SHORT[r % len(SHORT)]); prof.append(PROFILES[(r // len(SHORT)) % len(PROFILES)])
    ts_l, sd_l = [], []
    for n, p in zip(counts, prof):
        t0 = float(torch.rand(1, generator=g)) * 2 + 2
        ts_l.append(t0 + DT * torch.arange(n, dtype=torch.float64)); sd_l.append(_profile(p, n, g))
    counts.append(2); prof.append("zeros")
    ts_l.append(torch.tensor([0.5, 60.0], dtype=torch.float64)); sd_l.append(torch.zeros(2, dtype=torch.float64))
    cnt = torch.tensor(counts)
    info = torch.stack([cnt.cumsum(0) - cnt, cnt], -1)
    ts = torch.cat(ts_l).float()
    te = (ts.double() + DT).float()
    dt = (te - ts).double()
    sigma = (torch.cat(sd_l) / dt).float()
    S = ts.shape[0]
    rgb = torch.rand(S, 3, generator=g)
    ri = torch.repeat_interleave(torch.arange(R), cnt)
    return dict(R=R, S=S, cnt=cnt, info=info, ts=ts, te=te, sigma=sigma, rgb=rgb, ri=ri, prof=prof, g=g,
                c=so.error_constant(cnt), dev={k: v.to(DEV) for k, v in
                                                 dict(info=info, ts=ts, te=te, sigma=sigma, rgb=rgb).items()})


def _check(name, got, ref, m, c, floor):
    """|got - ref| <= c U32 M + floor element-wise, and exactly 0 where M = 0."""
    got, ref = got.detach().cpu().double(), ref.double()
    err = (got - ref).abs()
    bound = c * so.U32 * m + floor
    bad = ~(err <= bound)
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {bad.numel()} outside the bound; worst err/bound "
                           f"{float((err / bound)[bad].max()):.3g}; first at {torch.nonzero(bad)[:5].flatten().tolist()}, "
                           f"got {got[bad][:5].tolist()} want {ref[bad][:5].tolist()}")
    zero = m == 0
    nz = zero & (got != 0)
    assert not nz.any(), (f"{name}: {int(nz.sum())} of {int(zero.sum())} entries with error scale 0 are not exactly 0, "
                          f"max |got| {float(got[nz].abs().max()):.3g}, first at {torch.nonzero(nz)[:5].flatten().tolist()}")
    return int(zero.sum())


def _sample_c(b):
    return b["c"][b["ri"]]


def test_composite_forward_within_float32_rounding_of_float64(batch):
    from nersemble_b200 import ops
    b, d = batch, batch["dev"]
    fwd = ops.composite(d["info"], d["ts"], d["te"], d["sigma"], d["rgb"], training=True)
    ref = so.composite(b["info"], b["ts"], b["te"], b["sigma"], b["rgb"])
    _check("weights", fwd["weights"][:, 0], ref["weights"], ref["weights_scale"], _sample_c(b), so.FLT_MIN)
    _check("rgb", fwd["rgb"], ref["rgb"], ref["rgb_scale"], b["c"][:, None], so.FLT_MIN)
    _check("accumulation", fwd["accumulation"][:, 0], ref["accumulation"], ref["accumulation_scale"], b["c"], so.FLT_MIN)
    _check("depth", fwd["depth"][:, 0], ref["depth"], ref["depth_scale"], b["c"], so.FLT_MIN)
    # the regimes are really there: denormal and zero weights, accumulation-0 rays clipped to the nearest midpoint
    w = fwd["weights"][:, 0].cpu()
    assert ((w > 0) & (w < so.FLT_MIN)).sum() > 100 and ((w == 0) & (ref["weights"] > 0)).sum() > 1000
    assert (fwd["accumulation"][:, 0].cpu()[b["cnt"] > 0] == 0).sum() > 100


@pytest.mark.parametrize("grads", ["all", "no_d_weights", "rgb_only"])
def test_composite_backward_within_float32_rounding_of_float64(batch, grads):
    from nersemble_b200 import ops
    b, d = batch, batch["dev"]
    g = torch.Generator().manual_seed(7)
    R, S = b["R"], b["S"]
    g_rgb = torch.randn(R, 3, generator=g) * 3
    g_acc = None if grads == "rgb_only" else torch.randn(R, generator=g) * 0.7
    g_dep = None if grads == "rgb_only" else torch.randn(R, generator=g) * 0.2
    g_w = torch.randn(S, generator=g) * 5 if grads == "all" else None
    dv = lambda x: None if x is None else x.to(DEV)
    fwd = ops.composite(d["info"], d["ts"], d["te"], d["sigma"], d["rgb"], training=True)
    args = (d["info"], d["ts"], d["te"], d["sigma"], d["rgb"], fwd["workspace"], g_rgb.to(DEV), dv(g_acc), dv(g_dep), dv(g_w))
    d_sigma, d_rgb = ops.composite_backward(*args)
    ref_s, ref_c, m_s, m_c = so.composite_backward(b["info"], b["ts"], b["te"], b["sigma"], b["rgb"], g_rgb, g_acc, g_dep, g_w)
    dt = (b["te"] - b["ts"]).double()
    c = _sample_c(b)
    n_zero = _check("d_sigma", d_sigma, ref_s, m_s, c, so.FLT_MIN * dt)
    _check("d_rgb", d_rgb, ref_c, m_c, c[:, None], so.FLT_MIN)
    assert n_zero > 100000, n_zero                      # occluded samples: exact zeros asserted, not just small
    # bitwise repeatable, and independent of where a ray lands in the launch: the rays in reverse order
    again = ops.composite_backward(*args)
    assert torch.equal(again[0], d_sigma) and torch.equal(again[1], d_rgb)
    flip = ops.composite_backward(d["info"].flip(0), *args[1:6], g_rgb.flip(0).to(DEV), dv(None if g_acc is None else g_acc.flip(0)),
                                  dv(None if g_dep is None else g_dep.flip(0)), dv(g_w))
    assert torch.equal(flip[0], d_sigma) and torch.equal(flip[1], d_rgb)


LOSS_CFG = dict(use_masked_rgb=True, alpha_mask_threshold=0.5, lambda_alpha=0.1, lambda_empty=0.5, lambda_near=0.25,
                lambda_depth=0.3, lambda_dist=0.02, eps_depth=0.35, dist_max_rays=2048)


def test_losses_within_float32_rounding_of_float64(batch):
    from nersemble_b200 import ops
    b, d = batch, batch["dev"]
    g = torch.Generator().manual_seed(8)
    R, S, info, cnt = b["R"], b["S"], b["info"], b["cnt"]
    fwd = ops.composite(d["info"], d["ts"], d["te"], d["sigma"], d["rgb"], training=True)
    w = fwd["weights"][:, 0].cpu()
    rgb, acc, depth = fwd["rgb"].cpu(), fwd["accumulation"][:, 0].cpu(), fwd["depth"][:, 0].cpu()
    image = torch.rand(R, 3, generator=g)
    alpha = torch.rand(R, generator=g); alpha[::3] = 1.0
    # depth targets a quarter dt off the sample grid, a quarter of the way into the ray (half the rays: none)
    first = b["ts"][info[:, 0].clamp(max=S - 1)].double()
    tgt = (first + ((cnt // 4) + 0.25) * DT).float() * (torch.arange(R) % 2 == 0)
    up = torch.tensor([0.5 + 0.37 * k for k in range(6)])
    vals, state = ops.losses_forward(d["info"], d["ts"], d["te"], fwd["weights"], fwd["rgb"], fwd["accumulation"],
                                     fwd["depth"], image.to(DEV), alpha.to(DEV), tgt.to(DEV), LOSS_CFG)
    d_rgb, d_acc, d_depth, d_w = ops.losses_backward(state, up.to(DEV))
    ref = so.losses(info, b["ts"], b["te"], w, rgb, acc, depth, image, alpha, tgt, LOSS_CFG, up)
    # the masks the kernels decide in float32 are the float64 ones (no midpoint near a threshold)
    mid32 = (b["ts"] + b["te"]) * 0.5
    t_s, eps = tgt[b["ri"]], torch.tensor(0.35)
    assert torch.equal((t_s > 0) & (t_s - eps <= mid32) & (mid32 <= t_s + eps), ref["masks"]["near"])
    assert torch.equal((t_s > 0) & (mid32 < t_s - eps), ref["masks"]["empty"])
    c = b["c"]
    _check("values", vals, ref["values"], ref["m_values"], c.max(), so.FLT_MIN)
    _check("d_rgb", d_rgb, ref["d_rgb"], ref["m_rgb"], c[:, None], so.FLT_MIN)
    _check("d_acc", d_acc, ref["d_acc"], ref["m_acc"], c, so.FLT_MIN)
    _check("d_depth", d_depth, ref["d_depth"], ref["m_depth"], c, so.FLT_MIN)
    n_zero = _check("d_weights", d_w, ref["d_weights"], ref["m_weights"], _sample_c(b), so.FLT_MIN)
    # the exact-zero case: rays at or beyond dist_max_rays, samples past the near band (no loss reads their weights)
    past = (b["ri"] >= LOSS_CFG["dist_max_rays"]) & (t_s > 0) & (mid32 > t_s + eps) & (w > 0)
    assert past.sum() > 1000 and (ref["m_weights"][past] == 0).all() and n_zero >= int(past.sum())
    assert ref["masks"]["near"].sum() > 10000 and ref["masks"]["empty"].sum() > 5000


@pytest.mark.parametrize("early_stop_eps,alpha_thre", [(1e-4, 1e-2), (0.0, 1e-2)])
def test_visibility_agrees_with_float64_away_from_the_thresholds(batch, early_stop_eps, alpha_thre):
    from nersemble_b200 import ops
    b, d = batch, batch["dev"]
    mask, kept = ops.visibility_mask(d["info"], d["ts"], d["te"], d["sigma"], early_stop_eps, alpha_thre)
    want, amb = so.visibility(b["info"], b["ts"], b["te"], b["sigma"], early_stop_eps, alpha_thre)
    mask = mask.cpu()
    flips = (mask != want) & ~amb
    assert not flips.any(), (int(flips.sum()), torch.nonzero(flips)[:5].flatten().tolist())
    assert int(amb.sum()) <= 1e-3 * b["S"] and 0 < int(want.sum()) < b["S"]
    # visibility_compact keeps exactly the samples of the mask, in order
    cand = {"t_starts": d["ts"], "t_ends": d["te"], "ray_indices": b["ri"].int().to(DEV), "packed_info": d["info"],
            "capacity": b["S"]}
    got = ops.visibility_compact(cand, d["sigma"], early_stop_eps, alpha_thre)
    k = int(got["n_total"].item())
    assert k == int(mask.sum()) and torch.equal(got["packed_info"][:, 1].cpu(), kept.cpu().long())
    assert torch.equal(got["t_starts"][:k].cpu(), b["ts"][mask]) and torch.equal(got["ray_indices"][:k].cpu(), b["ri"].int()[mask])
