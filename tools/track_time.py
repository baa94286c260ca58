"""Cost of point tracking on a config-2-sized model (bench.synthetic_params: full-size tables, T = 24), with CUDA events
(median of REPS calls after one warm-up):
  * the Jacobian pass (ops.deform_jacobian) over 1 M points;
  * the inverse (ops.deform_inverse) over the same 1 M points, tracked from one timestep to another (targets from the
    Jacobian pass's own offsets at the source time), with the iteration histogram and the convergence rate;
  * a mesh sequence over all 24 timesteps (ops.extract_mesh_sequence) at MESH_RES points along the longest axis, and
    its parts: the reference mesh, the tracking of its vertices and the per-frame vertex attributes.
Prints the card name and power limit of this run."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from nersemble_b200 import ops

dev = torch.device("cuda", 0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print("gpu:", torch.cuda.get_device_name(0), "|", smi[0] if smi else "nvidia-smi n/a")
REPS = int(os.environ.get("REPS", "5"))
MESH_RES = int(os.environ.get("MESH_RES", "96"))
N = 1 << 20
T0, T1, WH, WD = 5.0 / 23.0, 11.0 / 23.0, 32.0, 7.0


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


S = bench.synthetic_params()
P = bench.native_params(S, dev)
gen = torch.Generator(device=dev).manual_seed(0)
lo, hi = P.aabb[0].to(dev), P.aabb[1].to(dev)
pts = lo + (0.1 + 0.8 * torch.rand((N, 3), device=dev, generator=gen)) * (hi - lo)
t0 = torch.full((N,), T0, device=dev)
with torch.no_grad():
    t_jac, jac = timed(lambda: ops.deform_jacobian(P, window_deform=WD, positions=pts, sample_times=t0))
    jn = jac["jacobian"].norm(dim=(-2, -1))
    print(f"jacobian: {N} points {t_jac:.2f} ms ({t_jac * (1 << 20) / N:.2f} ms per 1 M points); |J|_F median "
          f"{jn.median().item():.3e}, max {jn.max().item():.3e}")
    targets = pts + jac["offsets"]
    t_inv, inv = timed(lambda: ops.deform_inverse(P, targets, uniform_time=T1, init=pts, window_deform=WD))
    hist = torch.bincount(inv["iterations"].long(), minlength=21).tolist()
    status = torch.bincount(inv["status"].long(), minlength=3).tolist()
    print(f"inverse {T0:.4f} -> {T1:.4f}: {N} points {t_inv:.2f} ms ({t_inv * (1 << 20) / N:.2f} ms per 1 M points); "
          f"converged {inv['converged'].float().mean().item():.6f}, status (converged, not, singular) {status}, "
          f"iterations histogram {hist}, moved median {(inv['positions'] - pts).norm(dim=-1).median().item():.3e}")
    t_same, same = timed(lambda: ops.deform_inverse(P, targets, uniform_time=T0, init=pts, window_deform=WD))
    print(f"inverse to the source time (0 iterations): {t_same:.2f} ms, iterations max {int(same['iterations'].max())}")
    del jac, inv, same, targets
    g = ops.density_grid(P, time=T0, resolution=MESH_RES, window_hash=WH, window_deform=WD)
    level = float(g["sigma"][1:-1, 1:-1, 1:-1].median())
    del g
    times = [t / 23.0 for t in range(24)]
    kw = dict(level=level, resolution=MESH_RES, window_hash=WH, window_deform=WD)
    t_seq, seq = timed(lambda: ops.extract_mesh_sequence(P, times=times, reference_time=T0, **kw), reps=max(1, REPS // 2))
    V, F = seq["vertices"].shape[1], seq["faces"].shape[0]
    t_ref, ref = timed(lambda: ops.extract_mesh(P, time=T0, normals=False, colours=False, **kw), reps=max(1, REPS // 2))
    v0 = ref["vertices"]
    t_trk, _ = timed(lambda: ops.track_points(P, v0, time_from=T0, times_to=times, window_deform=WD), reps=max(1, REPS // 2))
    print(f"mesh sequence, 24 timesteps, {MESH_RES}^3 grid: V {V}, F {F}: {t_seq:.1f} ms = reference mesh {t_ref:.1f} ms + "
          f"tracking {t_trk:.1f} ms + attributes {t_seq - t_ref - t_trk:.1f} ms (by difference); converged "
          f"{seq['converged'].float().mean().item():.6f}")
