"""Time the stages of the fused field kernel separately (CUDA events) to see where the time goes.
    python tools/kernel_sweep.py            (on an H100)"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from nersemble_b200 import ops

dev = torch.device("cuda", 0)
P = bench.native_params(bench.synthetic_params(), dev)
o, d, t = bench.synthetic_rays(bench.RAYS, 1000, dev)
ts, te, ri, info = ops.march_fixed(o, d, P.aabb, bench.SAMPLES_PER_RAY, bench.STEP, bench.NEAR)
n = ts.numel()


def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


kw = dict(origins=o, directions=d, ray_times=t, t_starts=ts, t_ends=te, ray_indices=ri)
res = {}
res["full(sigma,rgb,offsets)"] = timeit(lambda: ops.field_forward(P, window_hash=32.0, window_deform=7.0, want=("sigma", "rgb", "offsets"), **kw))
res["density_only(deform+hash+base)"] = timeit(lambda: ops.field_forward(P, window_hash=32.0, window_deform=7.0, want=("sigma",), **kw))
res["no_deform(hash+base+head)"] = timeit(lambda: ops.field_forward(P, window_hash=32.0, window_deform=None, use_deformation=False, want=("sigma", "rgb"), **kw))
res["no_deform_density(hash+base)"] = timeit(lambda: ops.field_forward(P, window_hash=32.0, window_deform=None, use_deformation=False, want=("sigma",), **kw))
res["offsets_only(deform)"] = timeit(lambda: ops.field_forward(P, window_hash=32.0, window_deform=7.0, want=("offsets",), **kw))
x = torch.rand((n, 3), device=dev); codes = torch.randn((n, 32), device=dev) * 0.2
res["hash_blend_kernel(random x)"] = timeit(lambda: ops.hash_blend_forward(P, x, codes, window_hash=32.0))
pos = (o[ri.long()] + d[ri.long()] * ((ts + te) / 2)[:, None])
xn = ((pos - P.aabb[0].to(dev)) / (P.aabb[1] - P.aabb[0]).to(dev)).clamp(0.001, 0.999).contiguous()
res["hash_blend_kernel(ray-ordered x)"] = timeit(lambda: ops.hash_blend_forward(P, xn, codes, window_hash=32.0))
f = ops.field_forward(P, window_hash=32.0, window_deform=7.0, want=("sigma", "rgb", "offsets"), **kw)
res["composite"] = timeit(lambda: ops.composite(info, ts, te, f["sigma"], f["rgb"], f["offsets"]))
res["march_fixed"] = timeit(lambda: ops.march_fixed(o, d, P.aabb, bench.SAMPLES_PER_RAY, bench.STEP, bench.NEAR))
for k, v in res.items():
    print(f"{k:40s} {v:8.3f} ms   {n / v / 1e3:8.1f} M samples/s   alg {16384 * n / v / 1e6:7.0f} GB/s")
print(json.dumps(res))
