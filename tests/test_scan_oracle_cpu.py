"""The float64 scan references of tests/scan_oracle.py against independent formulations: autograd through
oracle.tp.nerfacc_cpu in float64, and central differences of the losses."""
import torch

import scan_oracle as so
from oracle.tp import nerfacc_cpu

F64 = torch.float64


def _rays(seed, counts, dt=0.011):
    g = torch.Generator().manual_seed(seed)
    cnt = torch.tensor(counts)
    R, S = len(counts), int(cnt.sum())
    ri = torch.repeat_interleave(torch.arange(R), cnt)
    info = torch.stack([cnt.cumsum(0) - cnt, cnt], -1)
    k = torch.arange(S) - info[:, 0][ri]
    ts = ((torch.rand(R, generator=g, dtype=F64) * 2 + 3)[ri] + k * dt).float()
    te = (ts.double() + dt).float()
    return g, info, ri, ts, te


def test_composite_and_its_gradient_match_nerfacc_autograd_in_float64():
    g, info, ri, ts, te = _rays(1, [0, 1, 5, 33, 70, 2])
    R, S = info.shape[0], ts.shape[0]
    sigma = (torch.rand(S, generator=g) * 40).float()
    sigma[40] = 1e5                                                    # opaque (sd 1100): the second sample of ray 4
    rgb = torch.rand(S, 3, generator=g).float()
    g_rgb, g_acc, g_dep = (torch.randn(R, 3, generator=g), torch.randn(R, generator=g), torch.randn(R, generator=g))
    g_w = torch.randn(S, generator=g)
    s64, c64 = sigma.double().requires_grad_(True), rgb.double().requires_grad_(True)
    ts64, te64 = ts.double(), te.double()
    w = nerfacc_cpu.render_weight_from_density(ts64, te64, s64, info)[0]
    acc = nerfacc_cpu.accumulate_along_rays(w, None, ri, R)
    comp = nerfacc_cpu.accumulate_along_rays(w, c64, ri, R) + (1.0 - acc)
    mid = ((ts64 + te64) / 2)[:, None]
    depth = torch.clip(nerfacc_cpu.accumulate_along_rays(w, mid, ri, R) / (acc + 1e-10), mid.min(), mid.max())
    L = (comp * g_rgb).sum() + (acc[:, 0] * g_acc).sum() + (depth[:, 0] * g_dep).sum() + (w * g_w).sum()
    L.backward()

    fwd = so.composite(info, ts, te, sigma, rgb)
    torch.testing.assert_close(fwd["weights"], w.detach(), rtol=1e-12, atol=1e-15)
    torch.testing.assert_close(fwd["rgb"], comp.detach(), rtol=1e-12, atol=1e-15)
    torch.testing.assert_close(fwd["accumulation"], acc[:, 0].detach(), rtol=1e-12, atol=1e-15)
    torch.testing.assert_close(fwd["depth"], depth[:, 0].detach(), rtol=1e-12, atol=1e-12)
    d_sigma, d_rgb, m_sigma, m_rgb = so.composite_backward(info, ts, te, sigma, rgb, g_rgb, g_acc, g_dep, g_w)
    # nerfacc's exclusive sum subtracts a batch-wide float64 prefix: ~1e-16 of the batch total is its noise floor
    torch.testing.assert_close(d_sigma, s64.grad, rtol=1e-9, atol=1e-13)
    torch.testing.assert_close(d_rgb, c64.grad, rtol=1e-9, atol=1e-15)
    # M bounds the magnitude of the expression it scales; behind the opaque sample it and the gradient are exactly 0
    assert (d_sigma.abs() <= m_sigma * (1 + 1e-12)).all() and (d_rgb.abs() <= m_rgb * (1 + 1e-12)).all()
    behind = torch.arange(41, 109)                                     # the rest of ray 4
    assert (m_sigma[behind] == 0).all() and (d_sigma[behind] == 0).all() and (d_rgb[behind] == 0).all()
    assert m_sigma[40] == 0 and d_sigma[40] == 0                       # exp(-sd) and every later weight are 0
    assert (m_sigma[:40] > 0).all()


def _loss_batch(seed=2):
    g, info, ri, ts, te = _rays(seed, [0, 6, 40, 1, 25, 60, 9])
    R, S = info.shape[0], ts.shape[0]
    w = (torch.rand(S, generator=g) * 0.08).float()
    rgb, image = torch.rand(R, 3, generator=g).float(), torch.rand(R, 3, generator=g).float()
    acc, alpha = torch.rand(R, generator=g).float(), torch.rand(R, generator=g).float()
    alpha[1] = 1.0
    depth = (torch.rand(R, generator=g) * 2 + 3).float()
    # depth targets a quarter dt off the sample grid: no midpoint lies near a mask threshold
    tgt = (ts[info[:, 0].clamp(max=S - 1)].double() + (info[:, 1] // 3 + 0.25) * 0.011).float()
    tgt[3] = 0.0
    cfg = dict(use_masked_rgb=True, alpha_mask_threshold=0.3, lambda_alpha=0.1, lambda_empty=0.5, lambda_near=0.25,
               lambda_depth=0.3, lambda_dist=0.02, eps_depth=0.0935, dist_max_rays=5)
    up = torch.tensor([0.5 + 0.37 * k for k in range(6)])
    return info, ts, te, w, rgb, acc, depth, image, alpha, tgt, cfg, up


def test_loss_gradients_match_central_differences():
    info, ts, te, w, rgb, acc, depth, image, alpha, tgt, cfg, up = _loss_batch()
    ref = so.losses(info, ts, te, w, rgb, acc, depth, image, alpha, tgt, cfg, up)
    m = ref["masks"]
    assert all(int(m[k].sum()) > 0 for k in ("masked", "bg", "empty", "near", "depth"))
    assert (ref["values"] > 0).all()
    base = dict(w=w.double(), rgb=rgb.double(), acc=acc.double(), depth=depth.double())

    def L(**over):
        a = {**base, **over}
        return float((so.losses(info, ts, te, a["w"], a["rgb"], a["acc"], a["depth"], image, alpha, tgt, cfg, up)["values"]
                      * up.double()).sum())

    h = 1e-6
    g = torch.Generator().manual_seed(9)
    for name, grad in (("w", ref["d_weights"]), ("rgb", ref["d_rgb"]), ("acc", ref["d_acc"]), ("depth", ref["d_depth"])):
        x = base[name].reshape(-1)
        for j in torch.randperm(x.numel(), generator=g)[:12].tolist():
            xp, xm = x.clone(), x.clone()
            xp[j] += h; xm[j] -= h
            fd = (L(**{name: xp.reshape(base[name].shape)}) - L(**{name: xm.reshape(base[name].shape)})) / (2 * h)
            got = float(grad.reshape(-1)[j])
            assert abs(fd - got) <= 1e-6 * max(1.0, abs(got)), (name, j, fd, got)


def test_loss_gradient_scales_bound_the_gradients_and_vanish_where_no_loss_reads_a_weight():
    info, ts, te, w, rgb, acc, depth, image, alpha, tgt, cfg, up = _loss_batch(3)
    ref = so.losses(info, ts, te, w, rgb, acc, depth, image, alpha, tgt, cfg, up)
    for k in ("weights", "rgb", "acc", "depth"):
        assert (ref["d_" + k].abs() <= ref["m_" + k] * (1 + 1e-12)).all(), k
    assert (ref["values"].abs() <= ref["m_values"] * (1 + 1e-12)).all()
    # ray 5 lies beyond dist_max_rays: its samples past the near band feed no loss
    s0, n = int(info[5, 0]), int(info[5, 1])
    mid = (ts.double() + te.double()) / 2
    past = torch.arange(s0, s0 + n)[mid[s0:s0 + n] > float(tgt[5]) + cfg["eps_depth"]]
    assert past.numel() > 5
    assert (ref["m_weights"][past] == 0).all() and (ref["d_weights"][past] == 0).all()


def test_visibility_matches_nerfacc_in_float64():
    g, info, ri, ts, te = _rays(4, [3, 0, 50, 200, 31])
    sigma = (torch.rand(ts.shape[0], generator=g) * 30).float()
    want = nerfacc_cpu.render_visibility_from_density(ts.double(), te.double(), sigma.double(), packed_info=info,
                                                      early_stop_eps=1e-3, alpha_thre=5e-2)
    vis, amb = so.visibility(info, ts, te, sigma, 1e-3, 5e-2)
    assert torch.equal(vis[~amb], want[~amb]) and amb.sum() <= 2 and vis.any() and (~vis).any()
