"""Host-side parameter layout for the CUDA kernels (pure torch ops; runs on CPU or GPU).

* hash tables: 8 tcnn grids (flat [(entry)*8 + p*2 + f], the reference's
  `field.hash_ensemble.hash_encodings.{c}.params`) <-> native [entry][member=c*4+p][feat] fp16,
  one 128-byte line per entry (field_components/hash_ensemble.py:102-112).
* MLP weights: nn.Linear / tcnn [out,in] matrices -> fp16 in mma.sync m16n8k16 B-fragment order,
  so a warp reads the fragments of two n-tiles with one 512-byte LDS.128 (csrc/nsb_field.cu).
* level table: tcnn's float32 formulas (grid.h) evaluated once on the host.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np
import torch

N_FREQ = 7
WARP_CODE_DIM = 128
DEFORM_IN_DIM = 3 * N_FREQ * 2 + 3 + WARP_CODE_DIM      # 173
DEFORM_IN_PAD = 48 + WARP_CODE_DIM                      # 176 (posenc permuted+padded to 48)


# ------------------------------------------------------------------ level table
def level_table(n_levels=16, log2_hashmap_size=19, base_resolution=16, per_level_scale=1.4472692012786865):
    """tcnn grid.h: scale = exp2f(l*log2f(s))*base - 1 (float32), res = ceil(scale)+1,
    entries = min(round_up(res^3, 8), 2^log2T); hashed iff entries < res^3-stride walk."""
    s = np.float32(per_level_scale)
    l2 = np.log2(s)
    out = dict(scale=[], res=[], entries=[], offset=[], hashed=[])
    off = 0
    for l in range(n_levels):
        sc = np.float32(np.exp2(np.float32(l) * l2) * np.float32(base_resolution) - np.float32(1.0))
        r = int(np.ceil(sc)) + 1
        e = min(((r ** 3 + 7) // 8) * 8, 1 << log2_hashmap_size)
        stride = 1
        for _ in range(3):
            if stride <= e:
                stride *= r
        out["scale"].append(float(sc)); out["res"].append(r); out["entries"].append(e)
        out["offset"].append(off); out["hashed"].append(int(e < stride))
        off += e
    out["total_entries"] = off
    out["n_levels"] = n_levels
    return out


# ------------------------------------------------------------------ hash tables
def tables_from_tcnn(grid_params: Sequence[torch.Tensor], n_feats: int = 2) -> torch.Tensor:
    """8 flat tcnn grids -> native [entries, 32, 2] (same dtype)."""
    P = 8 // n_feats
    per = [g.reshape(-1, P, n_feats) for g in grid_params]
    return torch.stack(per, 1).reshape(per[0].shape[0], len(per) * P, n_feats).contiguous()


def tables_to_tcnn(tables: torch.Tensor) -> List[torch.Tensor]:
    N, H, F = tables.shape
    P = 8 // F
    t = tables.reshape(N, H // P, P, F)
    return [t[:, c].reshape(-1).contiguous() for c in range(H // P)]


# ------------------------------------------------------------------ MMA B-fragment packing
def _f(t: torch.Tensor) -> torch.Tensor:
    """fp32 view of a weight -- or the tensor itself when it carries int64 element ids (gather-plan tracing)."""
    return t if t.dtype == torch.int64 else t.detach().float()


def pack_mma_b(W: torch.Tensor, colmap: Sequence[int], group_cols: int) -> torch.Tensor:
    """W [N_out, K_in] -> fp16 tensor in order [group][k-tile][n-tile pair][lane][ntsel][hi][e]:
    lane = g*4+q holds, for n = group*group_cols + pair*16 + ntsel*8 + g and
    k = kt*16 + hi*8 + 2q + e, the element W[n, colmap[k]] (0 where colmap[k] < 0 or n >= N_out)."""
    N, _ = W.shape
    Kp = len(colmap)
    assert Kp % 16 == 0 and group_cols % 16 == 0
    Np = ((N + group_cols - 1) // group_cols) * group_cols
    cm = torch.as_tensor(list(colmap), dtype=torch.long, device=W.device)
    ids = W.dtype == torch.int64                     # gather-plan tracing (gather_plan below): element ids, 0 = zero
    Wp = torch.zeros((Np, Kp), dtype=torch.int64 if ids else torch.float32, device=W.device)
    valid = cm >= 0
    Wp[:N][:, valid] = _f(W)[:, cm[valid]]
    Wh = Wp if ids else Wp.half()
    G, NPR, KT = Np // group_cols, group_cols // 16, Kp // 16
    t = Wh.view(G, NPR, 2, 8, KT, 2, 4, 2)          # (grp, pair, ntsel, g, kt, hi, q, e)
    t = t.permute(0, 4, 1, 3, 6, 2, 5, 7)           # (grp, kt, pair, g, q, ntsel, hi, e)
    return t.contiguous().view(-1)


def deform_input_colmap() -> List[int]:
    """Kernel input column k' (176) -> reference input column (173) of mlp_stem layer 0.
    Kernel order: pairs (sin, cos) of arg i = dim*7 + freq for i < 21, then (2pi x, 2pi y),
    (2pi z, 0), (0, 0), then the 128 warp-code columns.  Reference order
    (windowed_nerf_encoding.py:50-73): sin block (21), cos block (21), 2pi*xyz (3), code (128)."""
    m = []
    for kp in range(48):
        i, s = divmod(kp, 2)
        if i < 21:
            m.append(i if s == 0 else 21 + i)
        elif i == 21:
            m.append(42 if s == 0 else 43)
        elif i == 22:
            m.append(44 if s == 0 else -1)
        else:
            m.append(-1)
    m += [45 + k for k in range(WARP_CODE_DIM)]
    return m


def pack_deform(stem_w: Sequence[torch.Tensor], stem_b: Sequence[torch.Tensor], r_w, r_b, v_w, v_b):
    """mlp_stem (6 Linear, skip at 4: input [in(173) | hidden(128)]), mlp_r, mlp_v
    (field_components/deformation_field.py:50-75) -> (packed fp16 weights, fp32 bias[776])."""
    assert len(stem_w) == 6 and stem_w[0].shape == (128, DEFORM_IN_DIM) and stem_w[4].shape == (128, DEFORM_IN_DIM + 128)
    packed = _deform_weights(stem_w, r_w, v_w, deform_input_colmap())
    bias = deform_bias_vector(stem_b, r_b, v_b)
    assert packed.numel() * 2 == 258048 and bias.numel() == 776
    return packed.contiguous(), bias


def pack_deform_tb(stem_w, stem_b, r_w, r_b, v_w, v_b, warp_codes: torch.Tensor):
    """Time-bias variant: the warp-code columns of layers 0 and 4 multiply a vector that only depends on the
    timestep, so W_code . code[t] + b is precomputed per timestep (fp16-rounded operands, fp32 accumulate -- the same
    products the MMA would form) and enters the kernel as a per-row bias.  Returns (packed fp16 without those
    columns, code_bias float [T,2,128])."""
    packed = _deform_weights(stem_w, r_w, v_w, deform_input_colmap()[:48])   # posenc part only (kernel order, padded to 48)
    assert packed.numel() * 2 == 94 * 2048
    return packed.contiguous(), deform_code_bias(stem_w, stem_b, warp_codes)


def pack_deform_bwd(stem_w, r_w, v_w) -> torch.Tensor:
    """Transposed weights for the delta GEMMs of nsb_deform_backward, in order of use:
    heads, L5, L4[:, hidden], L4[:, code], L3, L2, L1, L0[:, code]  (K = 128 outputs; N = 128 columns in two halves).
    Hidden columns of layer 4 are the reference columns 173.., code columns are 45..172 of layers 0 and 4."""
    o128 = list(range(128))
    heads = torch.cat([_f(v_w), _f(r_w)], 0)            # [6, 128]: rows = (v, r) outputs
    parts = [pack_mma_b(heads.t(), list(range(6)) + [-1] * 10, 64)]
    def T(w, cols):
        return pack_mma_b(_f(w)[:, cols].t(), o128, 64)
    code = list(range(45, DEFORM_IN_DIM))
    hidden4 = list(range(DEFORM_IN_DIM, DEFORM_IN_DIM + 128))
    parts += [T(stem_w[5], o128), T(stem_w[4], hidden4), T(stem_w[4], code), T(stem_w[3], o128), T(stem_w[2], o128),
              T(stem_w[1], o128), T(stem_w[0], code)]
    packed = torch.cat(parts)
    assert packed.numel() * 2 == 114 * 2048
    return packed.contiguous()


def pack_deform_pe_t(w0: torch.Tensor, w4: torch.Tensor) -> torch.Tensor:
    """Transposed posenc columns of stem layers 0 and 4 for nsb_deform_input_grad: two [K = 128 outputs -> N = 48] blocks
    (N in the kernel's posenc order, deform_input_colmap()[:48]; padding columns are zero), each in MMA-B fragment order
    with 3 n-tile pairs per k-tile.  pack_deform_bwd only carries the hidden and code columns."""
    cm = torch.as_tensor(deform_input_colmap()[:48], dtype=torch.long, device=w0.device)
    valid = cm >= 0
    parts = []
    for w in (w0, w4):
        wpe = torch.zeros((128, 48), dtype=torch.float32, device=w.device)
        wpe[:, valid] = _f(w)[:, cm[valid]]
        parts.append(pack_mma_b(wpe.t(), list(range(128)), 48))
    packed = torch.cat(parts)
    assert packed.numel() * 2 == 2 * 12288
    return packed.contiguous()


def head_input_colmap() -> List[int]:
    """Kernel colour-MLP input column -> reference column of [d'(3) | geo(15) | ones(14)]
    (fields/nersemble_nerfacto_field.py:371-377 + tcnn pad-with-1.0).  Kernel order:
    [1.0 | geo(15) | d'(3) | 1.0 x 13] so the density-MLP accumulators feed k-tile 0 directly."""
    return [18] + [3 + j for j in range(15)] + [0, 1, 2] + list(range(19, 32))


def pack_field(base_w: Sequence[torch.Tensor], head_w: Sequence[torch.Tensor]) -> torch.Tensor:
    """tcnn mlp_base (32->64->16) and mlp_head (32->64->64->16) weight matrices [out,in]."""
    assert base_w[0].shape == (64, 32) and base_w[1].shape == (16, 64)
    assert head_w[0].shape == (64, 32) and head_w[1].shape == (64, 64) and head_w[2].shape == (16, 64)
    parts = [pack_mma_b(base_w[0], range(32), 64), pack_mma_b(base_w[1], range(64), 16),
             pack_mma_b(head_w[0], head_input_colmap(), 64), pack_mma_b(head_w[1], range(64), 64),
             pack_mma_b(head_w[2], range(64), 16)]
    packed = torch.cat(parts)
    assert packed.numel() * 2 == 20480
    return packed.contiguous()


def pack_field_bwd(base_w: Sequence[torch.Tensor], head_w: Sequence[torch.Tensor]) -> torch.Tensor:
    """Transposed weights for the delta GEMMs dX = delta . W (K = out dim, N = in dim), same fragment order and
    the same per-layer offsets as pack_field.  Head layer 0 keeps the kernel's permuted input column order on N."""
    hm = head_input_colmap()
    parts = [pack_mma_b(base_w[0].t(), range(64), 32), pack_mma_b(base_w[1].t(), range(16), 64),
             pack_mma_b(head_w[0][:, hm].t(), range(64), 32), pack_mma_b(head_w[1].t(), range(64), 64),
             pack_mma_b(head_w[2].t(), range(16), 64)]
    packed = torch.cat(parts)
    assert packed.numel() * 2 == 20480 and [p.numel() // 8 for p in parts] == [256, 128, 256, 512, 128]
    return packed.contiguous()


# ------------------------------------------------------------------ gather plans
# Training re-packs the MLP weights every step (they change every step).  The packers above are the definition of the
# layouts but cost ~300 small torch ops per step (advanced indexing per layer: host time comparable to
# the GPU time of the forward).  A plan is the same packer traced once on int64 element ids: afterwards packing is
# cat(sources) -> one gather -> half.
_PLANS: dict = {}


def gather_plan(name: str, fn, shapes: Sequence[Sequence[int]], device) -> torch.Tensor:
    """Index tensor `idx` such that fn(*ws) == cat([0], *[w.reshape(-1) for w in ws])[idx].half() for weights of the
    given shapes.  fn must build its result from _f()/pack_mma_b/slicing/cat only."""
    key = (name, str(device))
    if key not in _PLANS:
        ids, ofs = [], 1
        for shp in shapes:
            n = 1
            for d in shp:
                n *= d
            ids.append(torch.arange(ofs, ofs + n, dtype=torch.int64, device=device).view(*shp))
            ofs += n
        idx = fn(*ids)
        assert idx.dtype == torch.int64
        _PLANS[key] = idx.contiguous()
    return _PLANS[key]


def apply_plan(idx: torch.Tensor, sources: Sequence[torch.Tensor]) -> torch.Tensor:
    flat = torch.cat([torch.zeros(1, dtype=torch.float32, device=idx.device)] + [_f(w).reshape(-1) for w in sources])
    return flat[idx].half()


_STEM_SHAPES = [(128, DEFORM_IN_DIM), (128, 128), (128, 128), (128, 128), (128, DEFORM_IN_DIM + 128), (128, 128)]
_FIELD_SHAPES = [(64, 32), (16, 64), (64, 32), (64, 64), (16, 64)]


def pack_deform_weights_fast(stem_w, r_w, v_w):
    """(pack_deform_tb weights, pack_deform_bwd) through cached gather plans."""
    dev = stem_w[0].device
    shapes = _STEM_SHAPES + [(3, 128), (3, 128)]
    src = list(stem_w) + [r_w, v_w]
    p_tb = gather_plan("deform_tb", lambda *w: _deform_weights(w[:6], w[6], w[7], deform_input_colmap()[:48]), shapes, dev)
    p_bwd = gather_plan("deform_bwd", lambda *w: pack_deform_bwd(w[:6], w[6], w[7]), shapes, dev)
    return apply_plan(p_tb, src), apply_plan(p_bwd, src)


def pack_field_fast(base_w, head_w):
    """(pack_field, pack_field_bwd) through cached gather plans."""
    dev = base_w[0].device
    src = list(base_w) + list(head_w)
    p_f = gather_plan("field", lambda *w: pack_field(w[:2], w[2:]), _FIELD_SHAPES, dev)
    p_b = gather_plan("field_bwd", lambda *w: pack_field_bwd(w[:2], w[2:]), _FIELD_SHAPES, dev)
    return apply_plan(p_f, src), apply_plan(p_b, src)


def pack_all_fast(stem_w, r_w, v_w, base_w, head_w):
    """All four packed weight buffers (pack_deform_tb weights, pack_deform_bwd, pack_field, pack_field_bwd) of a
    training step with ONE cat, ONE gather and ONE cast (host time: ~25 torch ops -> 3)."""
    dev = stem_w[0].device
    key = ("all", str(dev))
    if key not in _PLANS:
        d_shapes = _STEM_SHAPES + [(3, 128), (3, 128)]
        n_deform = sum(a * b for a, b in d_shapes)
        plans = [gather_plan("deform_tb", lambda *w: _deform_weights(w[:6], w[6], w[7], deform_input_colmap()[:48]), d_shapes, dev),
                 gather_plan("deform_bwd", lambda *w: pack_deform_bwd(w[:6], w[6], w[7]), d_shapes, dev)]
        f_plans = [gather_plan("field", lambda *w: pack_field(w[:2], w[2:]), _FIELD_SHAPES, dev),
                   gather_plan("field_bwd", lambda *w: pack_field_bwd(w[:2], w[2:]), _FIELD_SHAPES, dev)]
        # field ids start after the deformation sources in the common flat buffer (id 0 stays the zero slot)
        f_plans = [torch.where(p > 0, p + n_deform, p) for p in f_plans]
        sizes = [int(p.numel()) for p in plans + f_plans]
        _PLANS[key] = (torch.cat(plans + f_plans).contiguous(), sizes)
    idx, sizes = _PLANS[key]
    packed = apply_plan(idx, list(stem_w) + [r_w, v_w] + list(base_w) + list(head_w))
    return torch.split(packed, sizes)


def _umma_block(Wb: torch.Tensor) -> torch.Tensor:
    """[N, 64] (N % 8 == 0) -> the wgmma K-major no-swizzle core-matrix order: 8 x 8 fp16 core matrices (8 rows x 16 B),
    byte offset = (n / 8) * 1024 + (k / 8) * 128 + (n % 8) * 16 + (k % 8) * 2  (descriptor LBO = 128, SBO = 1024)."""
    N = Wb.shape[0]
    assert Wb.shape[1] == 64 and N % 8 == 0
    return Wb.reshape(N // 8, 8, 8, 8).permute(0, 2, 1, 3).contiguous().view(-1)


def _pad2(W: torch.Tensor, rows: int, cols: int) -> torch.Tensor:
    out = torch.zeros((rows, cols), dtype=W.dtype, device=W.device)
    out[:W.shape[0], :W.shape[1]] = W
    return out


def pack_deform_umma(stem_w, r_w, v_w) -> torch.Tensor:
    """Deformation weights for the wgmma tensor role (nsb_field_tensor_role_tc.inc): 14 blocks in order of use, each
    [n x 64 k] in core-matrix order (_umma_block).  K follows the reference's input column order
    (windowed_nerf_encoding.py:50-73: sin 21 | cos 21 | 2 pi p 3), zero-padded to 64; the 128 warp-code columns of
    layers 0 and 4 are not here (they enter as the per-timestep code bias, deform_code_bias):
      L0 [128 x 45->64] | L1, L2, L3 [128 x 64] x 2 each | L4 hidden (reference columns 173..300) x 2, posenc 45->64 |
      L5 x 2 | heads (rows v0..2, r0..2, zero to 16) x 2.   12 * 16 KB + 2 * 2 KB = 200704 bytes."""
    W = [_f(w) for w in stem_w]
    blocks = [_umma_block(_pad2(W[0][:, :45], 128, 64))]
    for l in (1, 2, 3):
        blocks += [_umma_block(W[l][:, :64]), _umma_block(W[l][:, 64:128])]
    h0 = DEFORM_IN_DIM
    blocks += [_umma_block(W[4][:, h0:h0 + 64]), _umma_block(W[4][:, h0 + 64:h0 + 128]), _umma_block(_pad2(W[4][:, :45], 128, 64))]
    blocks += [_umma_block(W[5][:, :64]), _umma_block(W[5][:, 64:128])]
    heads = _pad2(torch.cat([_f(v_w), _f(r_w)], 0), 16, 128)
    blocks += [_umma_block(heads[:, :64]), _umma_block(heads[:, 64:])]
    out = torch.cat(blocks)
    assert out.numel() * 2 == 12 * 16384 + 2 * 2048
    return out if out.dtype == torch.int64 else out.half().contiguous()


def pack_deform_umma_fast(stem_w, r_w, v_w) -> torch.Tensor:
    dev = stem_w[0].device
    plan = gather_plan("deform_umma", lambda *w: pack_deform_umma(w[:6], w[6], w[7]), _STEM_SHAPES + [(3, 128), (3, 128)], dev)
    return apply_plan(plan, list(stem_w) + [r_w, v_w])


def _deform_weights(stem_w, r_w, v_w, in_map):
    """The weight part shared by pack_deform (in_map = 176 columns) and pack_deform_tb (48 posenc columns)."""
    ident = list(range(128))
    skip_map = [DEFORM_IN_DIM + k for k in range(128)] + list(in_map)
    maps = [in_map, ident, ident, ident, skip_map, ident]
    parts = [pack_mma_b(w, m, 64) for w, m in zip(stem_w, maps)]
    parts.append(pack_mma_b(torch.cat([_f(v_w), _f(r_w)], 0), ident, 16))
    return torch.cat(parts)


def deform_bias_vector(stem_b, r_b, v_b) -> torch.Tensor:
    dev = stem_b[0].device
    return torch.cat([b.detach().float().reshape(-1) for b in stem_b] +
                     [v_b.detach().float().reshape(-1), r_b.detach().float().reshape(-1), torch.zeros(2, device=dev)]).contiguous()


def deform_code_bias(stem_w, stem_b, warp_codes: torch.Tensor) -> torch.Tensor:
    """[T, 2, 128]: W_code(layer 0 | 4) . warp_code[t] + bias (see pack_deform_tb)."""
    ch = warp_codes.detach().half().float()
    cb = []
    for l in (0, 4):
        wc = stem_w[l].detach()[:, 45:DEFORM_IN_DIM].half().float()
        cb.append(ch @ wc.t() + stem_b[l].detach().float()[None, :])
    return torch.stack(cb, 1).contiguous()


def split_tcnn_mlp_params(flat: torch.Tensor, shapes: Sequence[Sequence[int]]) -> List[torch.Tensor]:
    """tcnn Network .params (layers consecutive, each [out,in] row-major) -> list of matrices."""
    out, ofs = [], 0
    for (o, i) in shapes:
        out.append(flat[ofs:ofs + o * i].view(o, i)); ofs += o * i
    assert ofs == flat.numel()
    return out


# ------------------------------------------------------------------ windows / blend folding
def posenc_window(windows_param: float, min_bands: float, max_bands: float, dim: int) -> torch.Tensor:
    """hash_ensemble.py:12-28 / windowed_nerf_encoding.py:76-92."""
    bands = torch.linspace(min_bands, max_bands, dim)
    x = torch.clamp(windows_param - bands, 0, 1)
    return 0.5 * (1 - torch.cos(torch.pi * x))


def blend_fold(window_hash: Optional[float], n_members: int = 32, disable_initial: bool = True,
               soft_transition: bool = True):
    """Fold hash_ensemble.py:119-139 into cw[h] = code[h]*scale[h] + bias[h]."""
    scale = torch.ones(n_members); bias = torch.zeros(n_members)
    if window_hash is not None:
        window = posenc_window(window_hash, 0, n_members - 1, n_members)
        if window_hash == 1 and disable_initial:
            scale = torch.zeros(n_members); bias = window.clone()
        elif soft_transition and window_hash < 2:
            alpha = window_hash - 1
            scale = window * alpha
            bias = torch.zeros(n_members); bias[0] = window[0] * (1 - alpha)
        else:
            scale = window
    return scale.tolist(), bias.tolist()


def deform_window(window_deform: Optional[float]) -> List[float]:
    if window_deform is None:
        return [1.0] * 8
    return posenc_window(window_deform, 0.0, N_FREQ - 1, N_FREQ).tolist() + [0.0]
