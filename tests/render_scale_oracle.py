"""Host-side helpers of tests/test_gpu_render_scale.py, device-agnostic and checked on the CPU by
tests/test_render_scale_oracle_cpu.py:

  * the persistent render kernels' tile schedule: packed sample s is row s % 128 of tile s // 128, and CTA c of a grid
    of `sms` CTAs runs tiles c, c + sms, c + 2 sms, ... (nsb_field_tensor_role_tc.inc: tile = blockIdx.x + it * gridDim.x),
    so tile k runs on CTA k % sms as that CTA's iteration k // sms;
  * a search for ragged batches (a chosen number of rows in the last tile, a chosen tile count modulo the grid);
  * the chunker that splits a batch into consecutive ray ranges of at most a given number of samples;
  * the eval-mode float64 composite (RGB with nan_to_num, white background and clamp, accumulation, expected depth with
    the global clip, the deformation renderer) with float32 error scales, on top of scan_oracle.composite;
  * reference-side mutations that model pipeline bugs (a stale tile buffer, rows shifted by one)."""
import math
from typing import List, Optional, Sequence, Tuple

import torch

import scan_oracle as so

TILE = 128          # NSB_TILE: rows per tile of the field phase


def n_tiles(n_samples: int) -> int:
    return (int(n_samples) + TILE - 1) // TILE


def tiles_per_cta(n_samples: int, sms: int) -> List[int]:
    """my_tiles of every CTA: (n_tiles - c + sms - 1) // sms, 0 for a CTA past the last tile."""
    nt = n_tiles(n_samples)
    return [(nt - c + sms - 1) // sms if c < nt else 0 for c in range(sms)]


def tile_place(tile: int, sms: int) -> Tuple[int, int]:
    """(CTA, iteration) of a tile."""
    return tile % sms, tile // sms


def tile_of(cta: int, it: int, sms: int) -> int:
    return cta + it * sms


def last_tile_rows(n_samples: int) -> int:
    """Rows of the last tile (0 for an empty batch)."""
    return (int(n_samples) - 1) % TILE + 1 if n_samples > 0 else 0


def ragged_batch(sms: int, last_rows: int, tiles_mod: int, per_ray: Sequence[int], min_tiles_per_cta: int = 8):
    """The smallest fixed-stride batch (R rays x S samples, S from `per_ray`) with at least min_tiles_per_cta tiles per
    CTA, whose last tile has `last_rows` rows and whose tile count is tiles_mod modulo sms.  Returns (R, S)."""
    best = None
    for S in per_ray:
        r0 = -(-min_tiles_per_cta * sms * TILE // S)
        for R in range(r0, r0 + TILE * sms):
            n = R * S
            if last_tile_rows(n) == last_rows and n_tiles(n) % sms == tiles_mod % sms:
                if best is None or n < best[0] * best[1]:
                    best = (R, S)
                break
    if best is None:
        raise ValueError(f"no batch with {last_rows} rows in the last tile and n_tiles = {tiles_mod} mod {sms}")
    return best


def chunk_rays(counts: torch.Tensor, max_samples: int) -> List[Tuple[int, int]]:
    """Consecutive ray ranges [a, b), greedy, each holding at most max_samples samples (and at least one ray)."""
    counts = [int(c) for c in counts.reshape(-1).tolist()]
    out, a, acc = [], 0, 0
    for r, c in enumerate(counts):
        if c > max_samples:
            raise ValueError(f"ray {r} has {c} samples, more than a chunk holds ({max_samples})")
        if acc + c > max_samples:
            out.append((a, r)); a, acc = r, 0
        acc += c
    if a < len(counts):
        out.append((a, len(counts)))
    return out


def probe_tiles(n_samples: int, sms: int, n_spread: int = 8) -> List[Tuple[str, int]]:
    """The tiles the small tests never reach, in priority order, as (label, tile): the ragged last tile; iterations 2
    and 3 (the first reuse of each of the two buffers) and the last two iterations of CTA 0, of a middle CTA and of the
    last CTA with work; then iterations 2 and 3 of n_spread CTAs spread over the grid."""
    nt = n_tiles(n_samples)
    mt = tiles_per_cta(n_samples, sms)
    busy = [c for c in range(sms) if mt[c] > 0]
    last = busy[-1]
    ctas = [0, last // 2, last]
    out, seen = [], set()

    def add(label, cta, it):
        if 0 <= it < mt[cta]:
            t = tile_of(cta, it, sms)
            if t not in seen:
                seen.add(t); out.append((label, t))
    lc, li = tile_place(nt - 1, sms)
    add("ragged last tile", lc, li)
    for c in ctas:
        for it in (2, 3):
            add(f"CTA {c} it {it}", c, it)
        for it in (mt[c] - 2, mt[c] - 1):
            add(f"CTA {c} it {it} (last two)", c, it)
    for k in range(n_spread):
        c = busy[(k * (len(busy) - 1)) // max(n_spread - 1, 1)]
        for it in (2, 3):
            add(f"CTA {c} it {it}", c, it)
    return out


def select_rays(ray_indices: torch.Tensor, tiles: Sequence[Tuple[str, int]], max_rays: int,
                extra: Sequence[int] = ()) -> Tuple[torch.Tensor, List[Tuple[str, int]]]:
    """The rays with samples in the given tiles, taking whole tiles in order while at most max_rays rays are chosen,
    plus the `extra` rays.  Returns (sorted ray ids, the tiles taken)."""
    ri = ray_indices.reshape(-1).long().cpu()
    chosen = set(int(r) for r in extra)
    taken = []
    for label, t in tiles:
        rays = set(torch.unique(ri[t * TILE:(t + 1) * TILE]).tolist())
        if len(chosen | rays) > max_rays:
            continue
        chosen |= rays; taken.append((label, t))
    return torch.tensor(sorted(chosen), dtype=torch.long), taken


def subset_samples(packed_info: torch.Tensor, rays: torch.Tensor):
    """Sample indices of `rays` (in ray order) and the packed_info / local ray index of the sub-batch."""
    info = packed_info.detach().cpu().long()
    start, cnt = info[rays, 0], info[rays, 1]
    idx = torch.cat([torch.arange(int(s), int(s) + int(c)) for s, c in zip(start, cnt)]) if rays.numel() else torch.zeros(0, dtype=torch.long)
    sub_cnt = cnt
    sub_info = torch.stack([torch.cumsum(sub_cnt, 0) - sub_cnt, sub_cnt], -1)
    local = torch.repeat_interleave(torch.arange(rays.numel()), sub_cnt)
    return idx, sub_info, local


def ordered_to_float(u: int) -> float:
    """nsb_common.cuh ordered_to_float of a uint32."""
    import struct
    u &= 0xffffffff
    bits = (u & 0x7fffffff) if (u & 0x80000000) else (~u & 0xffffffff)
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def midpoint_range(t_starts: torch.Tensor, t_ends: torch.Tensor) -> Optional[Tuple[float, float]]:
    """min / max of the float32 midpoints (t_start + t_end) / 2, as composite_ray computes them (None: no sample)."""
    if t_starts.numel() == 0:
        return None
    mid = (t_starts.float() + t_ends.float()) / 2
    return float(mid.min()), float(mid.max())


def composite_eval(packed_info, t_starts, t_ends, sigma, rgb, offsets=None, clip=None):
    """Eval-mode composite in float64 (RGBRenderer: nan_to_num of the sample colours, white background, clamp to [0, 1];
    AccumulationRenderer; DepthRenderer('expected') clipped to `clip` (default: the float64 range of the midpoints);
    the deformation renderer), each output with its float32 error scale *_scale as in scan_oracle:
    |x32 - x64| <= error_constant(n) U32 scale.  Clamping and clipping are 1-Lipschitz and keep the bound."""
    rgb32 = torch.nan_to_num(rgb.detach().float().cpu(), nan=0.0)          # +-inf -> +-FLT_MAX, as the kernel does
    out = so.composite(packed_info, t_starts, t_ends, sigma, rgb32)
    out["rgb"] = out["rgb"].clamp(0.0, 1.0)
    if clip is not None:
        out["clip"] = clip
        out["depth"] = out["draw"].clamp(*clip)
    if offsets is not None:
        off = offsets.detach().cpu().double()
        R = packed_info.shape[0]
        d, ds = torch.zeros(R, 3, dtype=so.F64), torch.zeros(R, 3, dtype=so.F64)
        for rays, idx in so._groups(packed_info):
            w, ws = out["weights"][idx], out["weights_scale"][idx]
            d[rays] = (w[..., None] * off[idx]).sum(1)
            ds[rays] = (ws[..., None] * off[idx].abs()).sum(1)
        out["deformation"], out["deformation_scale"] = d, ds
    return out


def stale_tile(values: torch.Tensor, tile: int, sms: int, n_samples: int) -> torch.Tensor:
    """A copy of per-sample `values` in which `tile` holds the values of the tile two iterations earlier on the same
    CTA (the previous user of its buffer), over the rows both tiles have."""
    src = tile - 2 * sms
    assert src >= 0, "the tile has no earlier user of its buffer"
    a, b = tile * TILE, min((tile + 1) * TILE, n_samples)
    out = values.clone()
    out[a:b] = values[src * TILE:src * TILE + (b - a)]
    return out


def shift_tile_rows(values: torch.Tensor, tile: int, n_samples: int) -> torch.Tensor:
    """A copy of per-sample `values` in which row i of `tile` holds row i + 1 (the last row keeps its own)."""
    a, b = tile * TILE, min((tile + 1) * TILE, n_samples)
    out = values.clone()
    out[a:b - 1] = values[a + 1:b]
    return out


def bound_ratio(got: torch.Tensor, want: torch.Tensor, bound: torch.Tensor) -> float:
    """max |got - want| / bound (an element with a zero bound and a non-zero difference counts as infinite)."""
    assert got.shape == want.shape, (tuple(got.shape), tuple(want.shape))
    err = (got.detach().cpu().double() - want.detach().cpu().double()).abs()
    bound = bound.detach().cpu().double().expand_as(err)
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def tol_ratio(got: torch.Tensor, want: torch.Tensor, rtol: float, atol: float) -> float:
    """max |got - want| / (atol + rtol |want|): torch.testing.assert_close passes exactly where this is <= 1."""
    want = want.detach().cpu().double()
    return bound_ratio(got, want, atol + rtol * want.abs())
