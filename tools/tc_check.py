"""A/B of the wgmma deformation role (flag name "tcgen05") (field_kernel_tc) against the mma.sync role (field_kernel_ws) on the same samples:
max |diff| of sigma / rgb / offsets and the kernel time of both.  Run under `timeout` on an H100."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from nersemble_b200 import ops

dev = torch.device("cuda", 0)
S = bench.synthetic_params()
deform = dict(stem_w=S["stem_w"], stem_b=S["stem_b"], r_w=S["r_w"], r_b=S["r_b"], v_w=S["v_w"], v_b=S["v_b"])
mk = lambda tc: ops.NativeParams.build(tables=S["tables"], base_w=S["base_w"], head_w=S["head_w"], time_emb=S["time_emb"],
                                       aabb=S["aabb"], levels=S["levels"], deform=deform, time_emb_deform=S["time_emb_deform"],
                                       device=dev, tcgen05=tc)
P0, P1 = mk(False), mk(True)
n_rays = int(sys.argv[1]) if len(sys.argv) > 1 else bench.RAYS
o, d, t = bench.synthetic_rays(n_rays, 1000, dev)
ts, te, ri, info = ops.march_fixed(o, d, P0.aabb, bench.SAMPLES_PER_RAY, bench.STEP, bench.NEAR)
kw = dict(origins=o, directions=d, ray_times=t, t_starts=ts, t_ends=te, ray_indices=ri)
want = ("sigma", "rgb", "offsets")
run = lambda P: ops.field_forward(P, window_hash=32.0, window_deform=7.0, want=want, **kw)
a = run(P0); torch.cuda.synchronize()
print("mma.sync role done", flush=True)
b = run(P1); torch.cuda.synchronize()
print("tcgen05 role done", flush=True)
for k in want:
    x, y = a[k].float(), b[k].float()
    print(f"{k:8s} max|diff| {float((x - y).abs().max()):.3e}   max|ref| {float(x.abs().max()):.3e}   nan {int(torch.isnan(y).sum())}")

def timeit(fn, reps=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps
print(f"field kernel ms ({ts.numel()} samples): mma.sync {timeit(lambda: run(P0)):.3f}   tcgen05 {timeit(lambda: run(P1)):.3f}")

# camera-frame case: ONE timestep for all rays -> per-frame blended table (NativeParams.frame_table) vs the per-sample blend
tu = torch.full_like(t, 0.5)
kwu = dict(kw, ray_times=tu)
per = ops.field_forward(P1, window_hash=32.0, window_deform=7.0, want=want, **kwu)
P1.frame_table(0.5, 32.0, True, True); torch.cuda.synchronize()
e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
P1._frame = None
e0.record(); P1.frame_table(0.5, 32.0, True, True); e1.record(); torch.cuda.synchronize()
print(f"nsb_blend_tables (one pass over the tables): {e0.elapsed_time(e1):.3f} ms")
fr = ops.field_forward(P1, window_hash=32.0, window_deform=7.0, want=want, uniform_time=0.5, **kwu)
for k in want:
    x, y = per[k].float(), fr[k].float()
    print(f"frame {k:8s} max|diff| {float((x - y).abs().max()):.3e}   max|ref| {float(x.abs().max()):.3e}")
tp = timeit(lambda: ops.field_forward(P1, window_hash=32.0, window_deform=7.0, want=want, **kwu))
tf = timeit(lambda: ops.field_forward(P1, window_hash=32.0, window_deform=7.0, want=want, uniform_time=0.5, **kwu))
print(f"uniform-time field kernel ms: per-sample blend {tp:.3f}   frame table {tf:.3f}")
