"""Torch oracle of the flow pass (DESIGN 4.2f): the sample selection of nsb_flow_select, the per-ray compositing of
nsb_flow_composite and the pinhole projection pi that inverts nsb_ray_batch's rays.  Selection is integer logic plus the
fp32 midpoint / target formation of the kernels (one rounding per operation, so it is compared exactly); compositing and
pi run in float64."""
import torch


def ray_directions(intrinsics, c2w, rows, cols):
    """Unnormalised-then-normalised world directions of pixels (row, col) as nsb_ray_batch builds them, in float64:
    d = R ((x - cx) / fx, -(y - cy) / fy, -1), x = col + 0.5, y = row + 0.5."""
    fx, fy, cx, cy = (float(v) for v in intrinsics)
    R = torch.as_tensor(c2w, dtype=torch.float64)[:3, :3]
    x, y = cols.double() + 0.5, rows.double() + 0.5
    dc = torch.stack([(x - cx) / fx, -(y - cy) / fy, -torch.ones_like(x)], -1)
    d = dc @ R.T
    return d / d.norm(dim=-1, keepdim=True)


def project(X, intrinsics, c2w):
    """pi(X) [n,2] (pixel x right, y down) and in_front [n]: Xc = R^T (X - o), x = cx + fx Xc.x / -Xc.z,
    y = cy - fy Xc.y / -Xc.z; in front iff -Xc.z > 0.  float64."""
    fx, fy, cx, cy = (float(v) for v in intrinsics)
    c = torch.as_tensor(c2w, dtype=torch.float64)
    Xc = (X.double() - c[:3, 3]) @ c[:3, :3]
    z = -Xc[:, 2]
    front = z > 0
    zs = torch.where(front, z, torch.ones_like(z))
    return torch.stack([cx + fx * Xc[:, 0] / zs, cy - fy * Xc[:, 1] / zs], -1), front


def select(packed_info, t_starts, t_ends, weights, offsets, origins, directions, n_total, min_weight):
    """nsb_flow_select: per ray, in order, the packed samples i < n_total of its segment with weights[i] >= min_weight.
    x = o + d (ts + te) / 2 and c = x + offset, formed in float32 with one rounding per operation like the kernels.
    Returns {"ray_sel" [R,2], "sel_index" [n], "targets" [n,3], "init" [n,3], "n_selected"}."""
    info = packed_info.cpu().long()
    w = weights.cpu().float().reshape(-1)
    ts, te = t_starts.cpu().float().reshape(-1), t_ends.cpu().float().reshape(-1)
    off = offsets.cpu().float().reshape(-1, 3)
    o, d = origins.cpu().float().reshape(-1, 3), directions.cpu().float().reshape(-1, 3)
    R = info.shape[0]
    n_total = min(int(n_total), w.shape[0])
    idx, ray, sel = [], [], torch.zeros((R, 2), dtype=torch.int64)
    for r in range(R):
        start, count = int(info[r, 0]), int(info[r, 1])
        seg = torch.arange(start, max(min(start + count, n_total), start), dtype=torch.int64)
        keep = seg[w[seg] >= min_weight] if seg.numel() else seg
        sel[r, 0], sel[r, 1] = len(idx), keep.numel()
        idx += keep.tolist()
        ray += [r] * keep.numel()
    idx_t, ray_t = torch.tensor(idx, dtype=torch.int64), torch.tensor(ray, dtype=torch.int64)
    mid = ts[idx_t] + te[idx_t]
    x = o[ray_t] + (d[ray_t] * mid[:, None]) * 0.5
    return {"ray_sel": sel, "sel_index": idx_t, "init": x, "targets": x + off[idx_t], "n_selected": len(idx)}


def composite(ray_sel, sel_index, init, positions, status, weights, camera=None):
    """nsb_flow_composite in float64: per ray, over its selected samples whose inverse converged (status 0),
    W = sum w, scene_flow = sum w (x' - x) / W (0 when W = 0); optical_flow = sum w (pi(x') - pi(x)) / sum w over those
    with both positions in front of the camera (0 when none).  camera: (intrinsics [4], camera_to_world [3,4])."""
    ray_sel = ray_sel.cpu().long()
    R = ray_sel.shape[0]
    n = int(ray_sel[:, 1].sum())
    idx = sel_index.cpu().long()[:n]
    x, y = init.cpu().double()[:n], positions.cpu().double()[:n]
    ok = status.cpu()[:n] == 0
    w = weights.cpu().double().reshape(-1)[idx] * ok
    ray = torch.repeat_interleave(torch.arange(R), ray_sel[:, 1])
    W = torch.zeros(R, dtype=torch.float64).index_add_(0, ray, w)
    S = torch.zeros((R, 3), dtype=torch.float64).index_add_(0, ray, w[:, None] * (y - x))
    out = {"flow_weight": W, "scene_flow": torch.where(W[:, None] > 0, S / W.clamp_min(1e-300)[:, None], torch.zeros_like(S))}
    if camera is not None:
        p0, f0 = project(x, *camera)
        p1, f1 = project(y, *camera)
        wp = w * (f0 & f1)
        Wp = torch.zeros(R, dtype=torch.float64).index_add_(0, ray, wp)
        F = torch.zeros((R, 2), dtype=torch.float64).index_add_(0, ray, wp[:, None] * (p1 - p0))
        out["optical_flow"] = torch.where(Wp[:, None] > 0, F / Wp.clamp_min(1e-300)[:, None], torch.zeros_like(F))
    return out
