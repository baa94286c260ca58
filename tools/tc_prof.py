"""Cycle breakdown of the wgmma deformation stage (debug build: tools/build_variant.sh tc_prof "-DNSB_TC_PROF",
run with NSB_LIB=tools/_variants/tc_prof.so): phases of thread 33 of CTA 3 (warpgroup 0, a row's sine / SE(3) thread),
per tile: the deformation of its 64 rows, then the density / colour MLPs of its warp's 16 rows."""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from nersemble_b200 import ops, _lib

dev = torch.device("cuda", 0)
P = bench.native_params(bench.synthetic_params(), dev)
o, d, t = bench.synthetic_rays(bench.RAYS, 1000, dev)
ts, te, ri, info = ops.march_fixed(o, d, P.aabb, bench.SAMPLES_PER_RAY, bench.STEP, bench.NEAR)
tu = torch.full_like(t, 0.5)
lib = _lib.load()
lib.nsb_debug_tc_prof.argtypes = [C.c_void_p]
names = ["feature wait + loop", "input loads", "posenc", "posenc barrier", "MMA completion (issue + wg_wait)",
         "epilogues, layers 1-3 and 5", "heads+SE3+xs", "density / colour MLPs", "epilogues, layers 0 and 4 (code bias)",
         "weight-ring wait (wait_blocks)"]
tiles = (ts.numel() // 128 + 131 - 3) // 132
for label, kw in (("per-sample blend", dict(ray_times=t)), ("frame table", dict(ray_times=tu, uniform_time=0.5)),
                  ("fused render kernel, fixed march, per-sample blend", None)):
    for _ in range(3):
        if kw is None:
            ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=bench.SAMPLES_PER_RAY,
                            near_plane=bench.NEAR, step=bench.STEP)
        else:
            ops.field_forward(P, window_hash=32.0, window_deform=7.0, want=("sigma", "rgb", "offsets"), origins=o, directions=d,
                              t_starts=ts, t_ends=te, ray_indices=ri, **kw)
    torch.cuda.synchronize()
    buf = (C.c_ulonglong * len(names))()
    assert lib.nsb_debug_tc_prof(buf) == 0
    tot = sum(buf)
    print(f"== {label}: {tiles} tiles on CTA 3, {tot / tiles:.0f} cycles per tile")
    for n_, v in zip(names, buf):
        print(f"   {n_:34s} {v / tiles:9.0f} cyc/tile  {100.0 * v / max(tot, 1):5.1f} %")

kb = (C.c_ulonglong * 8)()
lib.nsb_debug_tc_prof_kernel.argtypes = [C.c_void_p]
assert lib.nsb_debug_tc_prof_kernel(kb) == 0
names_k = ["setup", "sampler phase (+ grid barrier)", "field phase (role)", "composite phase"]
print("== render_kernel_tc, CTA 3, cycles between phase boundaries:")
for i, n_ in enumerate(names_k):
    print(f"   {n_:34s} {kb[i + 1] - kb[i]:10d}")
