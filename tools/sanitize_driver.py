"""Small end-to-end exercise of every libnsb kernel, sized for compute-sanitizer (tools/sanitize.sh):
fixed + occupancy march, visibility mask, fused field forward (inference and training instantiations, ragged last tile,
several tiles per CTA so the mbarrier ring / tile counters wrap), composite fwd/bwd, losses, field / deformation
backward, rank-1 expand + fused Adam, occupancy update, component kernels, surface normals (canonical and observation
space), the deformation input gradient (ragged last tile, a device sample count below the buffer size), the mesh export
(a ragged last tile of grid points, an occupancy grid, vertex normals and colours), the deformation Jacobian and inverse
(ragged last tile, several tiles per CTA, per-sample warp codes), a tracked mesh sequence, and the flow pass (selection
of a fixed-stride render, the inverse over the device-side selected count, compositing with a camera), and renders
between timesteps on both gathers."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import bench
from nersemble_b200 import ops
from nersemble_b200.nerfstudio_shim import RayBundle
from nersemble_b200.optim import FusedFieldsAdam

dev = torch.device("cuda", 0)
R = int(os.environ.get("SAN_RAYS", "160"))
S = bench.synthetic_params(n_timesteps=4, log2T=12)
P = bench.native_params(S, dev)
o, d, t = bench.synthetic_rays(R, 3, dev)
ts, te, ri, info = ops.march_fixed(o, d, P.aabb, 100, bench.STEP, bench.NEAR)          # 16 000 samples = 125 tiles
out = ops.render_packed(P, o, d, t, ts, te, ri, info, window_hash=32.0, window_deform=7.0, training=False)
out2 = ops.render_packed(P, o, d, t, ts[:-37], te[:-37], ri[:-37],
                         torch.stack([info[:, 0], torch.clamp(info[:, 1] - torch.tensor([0] * (R - 1) + [37], device=dev), min=0)], -1),
                         window_hash=1.5, window_deform=3.3, training=False)                 # ragged last tile
x = torch.rand((500, 3), device=dev); codes = torch.randn((500, 32), device=dev) * 0.2
ops.hash_blend_forward(P, x, codes, window_hash=20.25)
ops.field_normals(P, window_hash=20.25, positions=P.aabb[0].to(dev) + x * (P.aabb[1] - P.aabb[0]).to(dev), sample_blend_codes=codes)
for lg in (False, True):        # normals of the render's packed samples: timestep stack and line gather, per-ray composite
    ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=100, near_plane=bench.NEAR,
                    step=bench.STEP, line_gather=lg, want_normals=True)
    ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=100, near_plane=bench.NEAR,
                    step=bench.STEP, line_gather=lg, want_normals=True, normals_space="observation")
ops.deform_input_grad(P, torch.randn((ts.shape[0] - 37, 3), device=dev), window_deform=3.3, origins=o, directions=d, ray_times=t,
                      t_starts=ts[:-37], t_ends=te[:-37], ray_indices=ri[:-37],
                      n_samples_dev=torch.tensor([9000], dtype=torch.int64, device=dev))
ops.deform_input_grad(P, torch.randn((500, 3), device=dev), positions=P.aabb[0].to(dev) + x * (P.aabb[1] - P.aabb[0]).to(dev),
                      sample_warp_codes=torch.randn((500, 128), device=dev) * 0.1)
ops.field_forward(P, window_hash=32.0, window_deform=7.0, positions=P.aabb[0].to(dev) + x * (P.aabb[1] - P.aabb[0]).to(dev),
                  sample_times=torch.rand(500, device=dev), want=("sigma",))
ops.extract_mesh(P, time=0.5, level=0.5, resolution=(13, 11, 9), window_hash=32.0, window_deform=7.0,
                 binaries=torch.rand((1, 16, 16, 16), device=dev) > 0.3, aabbs=P.aabb.reshape(1, 6).to(dev))
xw = P.aabb[0].to(dev) + torch.rand((4100, 3), device=dev) * (P.aabb[1] - P.aabb[0]).to(dev)
tw = torch.rand(4100, device=dev)
ops.deform_jacobian(P, window_deform=3.3, positions=xw, sample_times=tw)
ops.deform_jacobian(P, positions=xw[:500], sample_warp_codes=torch.randn((500, 128), device=dev) * 0.1)
ops.deform_inverse(P, xw, sample_times=tw, window_deform=3.3, max_iter=5)
ops.track_points(P, xw[:77], time_from=0.25, times_to=[0.0, 1.0], window_deform=7.0)
ops.extract_mesh_sequence(P, times=[0.0, 1.0], reference_time=0.5, level=0.5, resolution=(13, 11, 9), window_hash=32.0,
                          window_deform=7.0)
cam = ((300.0, 310.0, 32.0, 24.0), torch.tensor([[1.0, 0.0, 0.0, 0.1], [0.0, 1.0, 0.0, 0.2], [0.0, 0.0, 1.0, 9.0]]))
rf = ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=100, near_plane=bench.NEAR,
                     step=bench.STEP)
ops.render_flow(P, rf, o, d, t, time_to=0.75, window_deform=7.0, camera=cam, max_iter=5)
ops.render_flow(P, rf, o, d, t, time_to=0.0, window_deform=7.0)
for lg in (False, True):        # renders between timesteps (nsb_render_forward_interp): timestep stack and line gather
    ops.render_rays(P, o, d, t, window_hash=32.0, window_deform=7.0, sampler="fixed", n_per_ray=100, near_plane=bench.NEAR,
                    step=bench.STEP, line_gather=lg, time_interpolation="linear")
# plugin model: occupancy march + pre-pass + training step + occupancy update
m = bench.build_model(S, dev).train()
occ = bench.blob_occupancy(seed=5)
m.occupancy_grid.binaries[0] = occ.to(dev); m.occupancy_grid.occs.copy_((occ.flatten().float() * 0.05).to(dev))
g = m.get_param_groups()
opts = [FusedFieldsAdam(g["fields"], lr=5e-3, eps=1e-15), torch.optim.Adam(g["embeddings"] + [p for p in g["deformation_field"] if p.requires_grad], lr=1e-3)]
rb = RayBundle(origins=o, directions=d, pixel_area=torch.ones(R, 1, device=dev),
               camera_indices=torch.zeros(R, 1, dtype=torch.long, device=dev), times=t)
gen = torch.Generator().manual_seed(0)
batch = {"image": torch.rand((R, 3), generator=gen).to(dev), "alpha_map": torch.randint(0, 256, (R, 1), generator=gen).float().to(dev),
         "depth_maps": (torch.rand(R, generator=gen) * 4 + 7).to(dev)}
for it in range(2):
    for op in opts:
        op.zero_grad()
    outs = m.get_outputs(rb)
    loss = sum(m.get_loss_dict(outs, batch).values())
    loss.backward()
    for op in opts:
        op.step()
m.get_training_callbacks(None)[0].run_callback(0)
m.get_training_callbacks(None)[0].run_callback(4096)
m.eval()
with torch.no_grad():
    m.get_outputs(rb)
torch.cuda.synchronize()
print("sanitize_driver: ok, loss", float(loss), "rgb mean", float(out["rgb"].mean()), float(out2["rgb"].mean()))
