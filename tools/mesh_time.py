"""Cost of the mesh export (ops.extract_mesh) for one timestep of a config-2-sized model (bench.synthetic_params:
full-size tables, T = 24), at 256^3 and 512^3 points along the longest axis, with the deformation (space="observation")
and without it (space="canonical").  Times each stage separately with CUDA events: the density pass (density_grid), the
extraction passes (marching_tetrahedra: count | scan | one host read of the totals | vertices | faces), the vertex normals
and the vertex colours.  For the extraction it reports the bytes the passes must move (counted from the grid and mesh
sizes, below) over its time.  Prints the card name and power limit of this run."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from nersemble_b200 import ops

dev = torch.device("cuda", 0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print("gpu:", torch.cuda.get_device_name(0), "|", smi[0] if smi else "nvidia-smi n/a")
REPS = int(os.environ.get("REPS", "3"))
TIME, WH, WD = 5.0 / 23.0, 32.0, 7.0


def timed(fn):
    """(median ms over REPS calls after one warm-up, last result)."""
    out = fn()
    ts = []
    for _ in range(REPS):
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2], out


def extraction_bytes(n_points, V, F):
    """Bytes the extraction passes move at least: count reads sigma (4 B) and writes the point mask (1 B); the vertex pass
    reads the mask and writes the vertex base (4 B) and the vertices (12 B each); the face pass reads mask and vertex
    base and writes the faces (12 B each)."""
    return n_points * (4 + 1 + 1 + 4 + 1 + 4) + 12 * (V + F)


S = bench.synthetic_params()
P = bench.native_params(S, dev)
kw = dict(time=TIME, window_hash=WH, window_deform=WD)
with torch.no_grad():
    for res in (256, 512):
        for space in ("observation", "canonical"):
            t_den, g = timed(lambda: ops.density_grid(P, resolution=res, space=space, **kw))
            sigma = g["sigma"]
            n = sigma.numel()
            level = float(sigma[1:-1, 1:-1, 1:-1].flatten()[:: max(1, n // (1 << 24))].median())
            t_ext, m = timed(lambda: ops.marching_tetrahedra(sigma, level, g["box_min"], g["h"]))
            V, F = m["vertices"].shape[0], m["faces"].shape[0]
            v = m["vertices"]
            vk = dict(positions=v, sample_times=torch.full((V,), TIME, device=dev), uniform_time=TIME, window_hash=WH)
            obs = space == "observation"

            def normals():
                o = ops.field_forward(P, window_deform=WD, want=("offsets",), **vk)["offsets"] if obs else None
                return ops.field_normals(P, offsets=o, world_space=True, space=space, window_deform=WD, **vk)["normals"]
            t_nrm, nrm = timed(normals)
            dirs = -nrm
            t_col, _ = timed(lambda: ops.field_forward(P, window_deform=WD, use_deformation=obs, sample_directions=dirs,
                                                        want=("rgb",), **vk)["rgb"])
            del sigma, g
            nb = extraction_bytes(n, V, F)
            nx, ny, nz = ops.mesh_grid(P, res)[2]
            print(f"{res}^3 {space}: grid {nx} x {ny} x {nz} = {n / 1e6:.1f} M points, "
                  f"level {level:.3g}, V {V}, F {F} | density {t_den:.2f} ms | extraction {t_ext:.2f} ms "
                  f"({nb / 1e9:.2f} GB, {nb / t_ext / 1e6:.0f} GB/s) | normals {t_nrm:.2f} ms | colours {t_col:.2f} ms "
                  f"(median of {REPS})")
            del m, v, nrm, dirs
            torch.cuda.empty_cache()
