"""Cost of the rendered normals channel (ops.render_rays(want_normals=True) / NeRSembleNGPModel.render_normals):
  config 2 shape: render_rays, fixed sampler, 4096 rays x 256 samples, T = 24 mixed timesteps (timestep stack), full-size
                  tables, with and without want_normals, alternating;
  config 4 frame: one camera frame through get_outputs_for_camera_ray_bundle (occupancy march of a head-sized blob,
                  uniform time -> frame table), render_normals off / on, alternating.
Each with no normals, canonical normals and observation-space normals (normals_space="observation": the canonical pass,
the deformation input gradient deform_input_grad_kernel and a combine pass), alternated in one process after warm-up.
Prints the card name and power limit of this run, the per-call times, each pass's share of the render time and the
tensor work of the input-gradient pass counted from shapes, and checks that the default outputs do not change with the
channel on."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from nersemble_b200 import ops
from nersemble_b200.nerfstudio_shim import RayBundle

dev = torch.device("cuda", 0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print("gpu:", torch.cuda.get_device_name(0), "|", smi[0] if smi else "nvidia-smi n/a")
REPS, ROUNDS = int(os.environ.get("REPS", "20")), int(os.environ.get("ROUNDS", "5"))


def timeit(fn, reps=REPS):
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


# MACs per sample of the input-gradient pass, from the layer shapes: the recomputed forward (posenc 48 -> 128, 4 x 128 -> 128,
# skip 176 -> 128, heads 128 -> 16 padded) and the delta chain (heads 16 -> 128, 5 x 128 -> 128, 2 x 128 -> 48 posenc)
VJP_FWD_MACS = 48 * 128 + 4 * 128 * 128 + 176 * 128 + 128 * 16
VJP_BWD_MACS = 16 * 128 + 5 * 128 * 128 + 2 * 128 * 48


def alternate(name, off, on, obs, n_samples):
    for _ in range(3):
        off(); on(); obs()
    t_off, t_on, t_obs = [], [], []
    for _ in range(ROUNDS):
        t_off.append(timeit(off)); t_on.append(timeit(on)); t_obs.append(timeit(obs))
    a, b, c = (sorted(t)[ROUNDS // 2] for t in (t_off, t_on, t_obs))
    flops = 2.0 * (VJP_FWD_MACS + VJP_BWD_MACS) * n_samples
    print(f"{name}: render {a:.3f} ms, with canonical normals {b:.3f} ms, with observation normals {c:.3f} ms (median of "
          f"{ROUNDS} alternating rounds of {REPS}); canonical pass +{b - a:.3f} ms = {100 * (b - a) / b:.1f} % of its render; "
          f"Jacobian passes +{c - b:.3f} ms = {100 * (c - b) / c:.1f} % of theirs; input-gradient tensor work "
          f"{flops / 1e9:.2f} GFLOP for {n_samples} samples = {flops / max(c - b, 1e-9) / 1e9:.1f} TFLOP/s over the added time")


S = bench.synthetic_params()
P = bench.native_params(S, dev)
R = bench.RAYS
o, d, t = bench.synthetic_rays(R, 1000, dev)
kw = dict(window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=bench.SAMPLES_PER_RAY, near_plane=bench.NEAR,
          step=bench.STEP)
with torch.no_grad():
    plain = ops.render_rays(P, o, d, t, **kw)
    withn = ops.render_rays(P, o, d, t, want_normals=True, **kw)
    for k in ("rgb", "accumulation", "depth", "deformation"):
        assert torch.equal(plain[k], withn[k]), k
    print("config2: timesteps in the batch", int(torch.unique((t.reshape(-1) * (S["time_emb"].shape[0] - 1)).round()).numel()),
          "| samples", int(plain["num_samples_per_ray"].sum()))
    alternate("config2 (4096 x 256, T=24 mixed)", lambda: ops.render_rays(P, o, d, t, **kw),
              lambda: ops.render_rays(P, o, d, t, want_normals=True, **kw),
              lambda: ops.render_rays(P, o, d, t, want_normals=True, normals_space="observation", **kw),
              int(plain["num_samples_per_ray"].sum()))

    # one config-4 camera frame
    H = W = int(os.environ.get("FRAME", "512"))
    model = bench.build_model(S, dev, eval_num_rays_per_chunk=1 << 19).eval()
    ax = (torch.arange(128, device=dev).float() + 0.5) / 128
    X, Y, Z = torch.meshgrid(ax, ax, ax, indexing="ij")
    model.occupancy_grid.binaries[0] = ((X - 0.5) ** 2 + (Y - 0.5) ** 2 + (Z - 0.5) ** 2) < 0.33 ** 2
    cam_o = torch.tensor([0.0, 0.0, 9.0], device=dev)
    ys, xs = torch.meshgrid(torch.linspace(0.25, -0.25, H, device=dev), torch.linspace(-0.25, 0.25, W, device=dev), indexing="ij")
    dd = torch.stack([xs, ys, -torch.ones_like(xs)], -1); dd = dd / dd.norm(dim=-1, keepdim=True)
    rb = RayBundle(origins=cam_o.expand(H, W, 3).contiguous(), directions=dd.contiguous(), pixel_area=torch.ones((H, W, 1), device=dev),
                   camera_indices=torch.zeros((H, W, 1), dtype=torch.long, device=dev), times=torch.full((H, W, 1), 5 / 23, device=dev))

    def frame(flag, space="canonical"):
        model.render_normals, model.render_normals_space = flag, space
        return model.get_outputs_for_camera_ray_bundle(rb)
    a, b = frame(False), frame(True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    print(f"config4 frame: {H}x{W}, samples", int(a["num_samples_per_ray"].sum()), "| rays with acc >= 0.5",
          int((b["accumulation"] >= 0.5).sum()))
    alternate(f"config4 frame ({H}x{W}, frame table)", lambda: frame(False), lambda: frame(True),
              lambda: frame(True, "observation"), int(a["num_samples_per_ray"].sum()))
