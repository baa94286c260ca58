"""Cost of rendering between timesteps (time_interpolation="linear", DESIGN 4.2g) against the nearest-timestep render,
on bench.synthetic_params (full-size tables), with CUDA events (median of REPS calls after one warm-up):
  * the config-2 shape: 4096 rays x 256 fixed-stride samples, T = 24, random continuous ray times, on the timestep stack;
  * the same with T = 48, on the line gather;
  * one H x W frame (default 512 x 512, occupancy sampler, blob grid, the bench's step) at an integer and at a fractional time, with the
    cached per-frame tables and with their build (the at_time view and its frame table) inside the timed call.
Prints the card name, power limit and maximum SM clock of this run."""
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from nersemble_b200 import ops

dev = torch.device("cuda", 0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print("gpu:", torch.cuda.get_device_name(0), "|", smi[0] if smi else "nvidia-smi n/a")
REPS = int(os.environ.get("REPS", "9"))
H = W = int(os.environ.get("FRAME", "512"))
WH, WD = 32.0, 7.0


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


def mixed(T, line_gather):
    S = bench.synthetic_params(n_timesteps=T)
    P = bench.native_params(S, dev)
    R, n_per = bench.RAYS, bench.SAMPLES_PER_RAY          # the config-2 batch, with continuous times
    o, d, _ = [x.to(dev) for x in bench.synthetic_rays(R, 1000)]
    t = torch.rand((R,), generator=torch.Generator().manual_seed(2)).to(dev)
    run = lambda mode: ops.render_rays(P, o, d, t, window_hash=WH, window_deform=WD, sampler="fixed", n_per_ray=n_per,
                                       near_plane=bench.NEAR, step=bench.STEP, line_gather=line_gather,
                                       time_interpolation=mode)
    with torch.no_grad():
        tn, _ = timed(lambda: run("nearest"))
        tl, _ = timed(lambda: run("linear"))
        tn2, _ = timed(lambda: run("nearest"))      # alternate: the spread between the two nearest runs is the noise
    shape = "line gather" if line_gather or P.timestep_tables(WH, True, True) is None else "timestep stack"
    print(f"mixed times, {R} rays x {n_per} samples, T = {T} ({shape}): nearest {tn:.3f} / {tn2:.3f} ms, "
          f"linear {tl:.3f} ms, linear / nearest {tl / min(tn, tn2):.3f}")
    del P
    torch.cuda.empty_cache()


def frame():
    S = bench.synthetic_params()
    P = bench.native_params(S, dev)
    T = P.n_timesteps
    fov = 0.36
    f = W / (2 * math.tan(fov / 2))
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32) + 0.5, torch.arange(W, dtype=torch.float32) + 0.5, indexing="ij")
    d = torch.stack([(xs - W / 2) / f, -(ys - H / 2) / f, -torch.ones_like(xs)], -1).reshape(-1, 3)
    d = (d / d.norm(dim=-1, keepdim=True)).to(dev)
    o = torch.tensor([0.0, 0.0, 9.0], device=dev).expand(H * W, 3).contiguous()
    R = H * W
    occ = bench.blob_occupancy().to(dev)[None]
    aabb = torch.tensor([float(v) for v in P.aabb_list], device=dev).reshape(1, 6)
    near, far = torch.full((R,), 0.2, device=dev), torch.full((R,), 1e3, device=dev)

    def run(t, mode, rebuild):
        if rebuild:
            P._frame = None; P._at_time = None
        return ops.render_rays(P, o, d, torch.full((R,), t, device=dev), window_hash=WH, window_deform=WD,
                               sampler="occupancy", near_planes=near, far_planes=far, binaries=occ, aabbs=aabb,
                               step=bench.STEP, uniform_time=t, time_interpolation=mode)
    ti, tf = 5 / (T - 1), 5.37 / (T - 1)
    with torch.no_grad():
        for rebuild in (False, True):
            a, ra = timed(lambda: run(ti, "nearest", rebuild))
            b, rb = timed(lambda: run(ti, "linear", rebuild))
            c, _ = timed(lambda: run(tf, "linear", rebuild))
            assert torch.equal(ra["rgb"], rb["rgb"])
            n = int(ra["_buffers"]["header"][2])
            print(f"frame {H} x {W} ({n} samples), {'with' if rebuild else 'without'} the table build: nearest at an "
                  f"integer time {a:.3f} ms, linear at an integer time {b:.3f} ms, linear at a fractional time {c:.3f} ms")


mixed(24, False)
mixed(48, False)
frame()
