"""Cost of the flow pass (ops.render_flow, DESIGN 4.2f) on a config-2-sized model (bench.synthetic_params: full-size
tables, T = 24) with the blob occupancy grid, for one camera frame of H x W pixels (default 512 x 512) at timestep 5,
flowed to timestep 11:
  * the frame rendered alone (get_outputs_for_camera_ray_bundle) against render + flow (render_flow), with CUDA events,
    median of REPS calls after one warm-up;
  * select, inverse and composite separately: kernel times from torch.profiler over one render_flow call of the frame,
    summed per stage;
  * the selected fraction of the packed samples, and the weight left out (accumulation - flow_weight), per frame.
The synthetic model is not a trained head: its densities are random and its warp barely moves between timesteps, so
the inverse mostly costs one Newton evaluation per tile.  Prints the card name and power limit of this run."""
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from nersemble_b200 import ops
from nersemble_b200.nerfstudio_shim import RayBundle

dev = torch.device("cuda", 0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print("gpu:", torch.cuda.get_device_name(0), "|", smi[0] if smi else "nvidia-smi n/a")
REPS = int(os.environ.get("REPS", "5"))
H = W = int(os.environ.get("FRAME", "512"))
T0, T1 = 5, 11


def timed(fn, reps=REPS):
    """(median ms over reps calls after one warm-up, last result)."""
    out = fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2], out


def camera(dist=9.0, azimuth=0.4, fov=0.36):
    """A pinhole on the bench's camera ring looking at the head volume: (intrinsics, camera_to_world [3,4])."""
    eye = torch.tensor([dist * math.sin(azimuth), 0.2, dist * math.cos(azimuth)], dtype=torch.float64)
    fwd = -eye / eye.norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64)); right = right / right.norm()
    up = torch.linalg.cross(right, fwd)
    f = W / (2 * math.tan(fov / 2))
    return (f, f, W / 2, H / 2), torch.cat([torch.stack([right, up, -fwd], -1), eye[:, None]], -1)


intr, c2w = camera()
ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64) + 0.5, torch.arange(W, dtype=torch.float64) + 0.5, indexing="ij")
dc = torch.stack([(xs - intr[2]) / intr[0], -(ys - intr[3]) / intr[1], -torch.ones_like(xs)], -1)
d = dc @ c2w[:, :3].T
d = (d / d.norm(dim=-1, keepdim=True)).float().to(dev)
o = c2w[:, 3].float().to(dev).expand(H, W, 3).contiguous()
S = bench.synthetic_params()
model = bench.build_model(S, dev).eval()
model.occupancy_grid.binaries[0] = bench.blob_occupancy().to(dev)
n_t = model.config.n_timesteps
bundle = RayBundle(origins=o, directions=d, pixel_area=torch.ones(H, W, 1, device=dev),
                   camera_indices=torch.zeros(H, W, 1, dtype=torch.long, device=dev),
                   times=torch.full((H, W, 1), T0 / (n_t - 1), device=dev))
cam = (torch.tensor(intr), c2w.float())

with torch.no_grad():
    t_render, img = timed(lambda: model.get_outputs_for_camera_ray_bundle(bundle))
    t_both, flow = timed(lambda: model.render_flow(bundle, T1, intrinsics=cam[0], camera_to_world=cam[1]))
    assert torch.equal(flow["rgb"], img["rgb"])
    print(f"frame {H} x {W} ({H * W} rays, {model.config.eval_num_rays_per_chunk} per chunk), timestep {T0} -> {T1}: "
          f"render {t_render:.2f} ms, render + flow {t_both:.2f} ms, flow {t_both - t_render:.2f} ms "
          f"({100 * (t_both - t_render) / t_render:.1f} % of the render)")

    # selection statistics, chunk by chunk as render_flow runs them
    P = model.native_params()
    _, wd = model._windows()
    n = model.config.eval_num_rays_per_chunk
    n_tot = n_sel = 0
    acc_sum = fw_sum = 0.0
    left = []
    for i in range(0, H * W, n):
        rb = bundle.get_row_major_sliced_ray_bundle(i, i + n)
        res = model._fused_render(rb, T0 / (n_t - 1))
        f = ops.render_flow(P, res, rb.origins.reshape(-1, 3), rb.directions.reshape(-1, 3), model._ray_times(rb),
                            time_to=T1 / (n_t - 1), window_deform=wd)
        n_tot += int(res["_buffers"]["header"][2]); n_sel += int(f["_n_selected"])
        acc_sum += float(res["accumulation"].sum()); fw_sum += float(f["flow_weight"].sum())
        left.append((res["accumulation"] - f["flow_weight"])[:, 0])
    left = torch.cat(left)
    covered = img["accumulation"].reshape(-1) > 0.5
    print(f"selection (min_weight {ops.FLOW_MIN_WEIGHT:g}): {n_sel} of {n_tot} packed samples ({100 * n_sel / max(n_tot, 1):.2f} %); "
          f"weight left out: {100 * (acc_sum - fw_sum) / max(acc_sum, 1e-30):.3f} % of the frame's accumulation, per ray "
          f"max {left.max().item():.3e}, mean {left.mean().item():.3e}, on rays with accumulation > 0.5 max "
          f"{left[covered].max().item() if covered.any() else 0.0:.3e}")
    conv = (flow["flow_weight"].sum() / flow["accumulation"].sum()).item()
    print(f"flow: |scene_flow| median {flow['scene_flow'].norm(dim=-1)[covered.view(H, W)].median().item():.3e} world units, "
          f"|optical_flow| median {flow['optical_flow'].norm(dim=-1)[covered.view(H, W)].median().item():.3e} px, "
          f"flow_weight / accumulation {conv:.5f}")

    # per-stage kernel times over one render_flow call of the frame
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.render_flow(bundle, T1, intrinsics=cam[0], camera_to_world=cam[1])
        torch.cuda.synchronize()
    stages = {"select": ("flow_count_kernel", "flow_scan_kernel", "flow_fill_kernel"), "inverse": ("deform_inv_kernel",),
              "composite": ("flow_composite_kernel",), "render": ("render_kernel", "march")}
    tot = {k: 0.0 for k in stages}
    for e in prof.key_averages():
        for k, names in stages.items():
            if any(s in e.key for s in names):
                tot[k] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0
                break
    print("kernel time per frame (torch.profiler): " + ", ".join(f"{k} {v:.2f} ms" for k, v in tot.items()))
