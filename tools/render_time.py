"""Times the inference render paths at BASELINE config 2 (4096 rays x 256 samples, full-size tables):
  3-kernel op path (march_fixed -> field_forward -> composite)      [5 launches]
  ops.render_rays fixed        (ONE launch)
  ops.render_rays occupancy    (cooperative march launch + one fused launch; all-ones grid, fars = 256 steps)
and checks that all three produce the same RGB."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from nersemble_b200 import ops
dev = torch.device("cuda", 0)
R = int(os.environ.get("RAYS", bench.RAYS))
P = bench.native_params(bench.synthetic_params(), dev)
o, d, t = bench.synthetic_rays(R, 1000, dev)
def timeit(fn, reps=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps
def three():
    ts, te, ri, info = ops.march_fixed(o, d, P.aabb, bench.SAMPLES_PER_RAY, bench.STEP, bench.NEAR)
    f = ops.field_forward(P, window_hash=32.0, window_deform=7.0, origins=o, directions=d, ray_times=t, t_starts=ts, t_ends=te, ray_indices=ri, want=("sigma", "rgb", "offsets"))
    return ops.composite(info, ts, te, f["sigma"], f["rgb"], f["offsets"], training=False)
def fixed():
    return ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=bench.SAMPLES_PER_RAY, near_plane=bench.NEAR, step=bench.STEP)
near = ops.march_fixed(o, d, P.aabb, 1, bench.STEP, bench.NEAR)[0]
far = near + bench.SAMPLES_PER_RAY * bench.STEP
occ = torch.ones((1, 128, 128, 128), dtype=torch.bool, device=dev)
aabbs = P.aabb.reshape(1, 6).to(dev)
def occupancy():
    return ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="occupancy", near_planes=near, far_planes=far, binaries=occ, aabbs=aabbs, step=bench.STEP, capacity=R * (bench.SAMPLES_PER_RAY + 2))
ref = three()["rgb"]
for name, fn in (("fixed", fixed), ("occupancy", occupancy)):
    out = fn(); torch.cuda.synchronize()
    print(name, "max |rgb - 3kernel|", float((out["rgb"] - ref).abs().max()), "n_total", int(out["_buffers"]["header"][2]))
print(f"ms: three_kernel {timeit(three):.3f}  fixed_1launch {timeit(fixed):.3f}  occupancy_2launch {timeit(occupancy):.3f}")
