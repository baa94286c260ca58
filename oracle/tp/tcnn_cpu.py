"""CPU restatement of the tiny-cuda-nn pieces the reference calls  [3P-mem].

TEST INFRASTRUCTURE (see oracle/__init__.py).  tiny-cuda-nn is an un-vendored,
unpinned git dependency of the reference (README.md:25-28, environment.yml:33-34);
its source is not on disk, so this file restates the published algorithm:

  * HashGrid encoding (include/tiny-cuda-nn/encodings/grid.h: grid_scale,
    grid_resolution, grid_index, kernel_grid; offset table in GridEncodingTemplated)
  * Identity encoding with pad-to-alignment by 1.0 (encodings/identity.h)
  * FullyFusedMLP / Network / NetworkWithInputEncoding (no bias, fp16 weights and
    activations, [out,in] row-major consecutive layers, output padded to 16)

Reference call sites: field_components/hash_ensemble.py:42-50,103;
fields/nersemble_nerfacto_field.py:99-112,137-153,162-172,285,322,377.

PARITY UNPINNED for this layer (no tcnn source / golden vectors available).
Everything is plain torch on CPU so autograd gives the backward oracle too.

Upstream map (tiny-cuda-nn master as of the reference's release, NVlabs/tiny-cuda-nn; a maintainer with the sources
can diff function by function):
  hashgrid_levels            include/tiny-cuda-nn/encodings/grid.h: GridEncodingTemplated ctor (offset table:
                             params_in_level = min(next_multiple(res^n, 8), 2^log2_hashmap_size)), grid_scale(),
                             grid_resolution()  [common_device.h in newer trees]
  hashgrid_indices_weights   grid.h: kernel_grid<T,N_POS_DIMS,N_FEATURES_PER_LEVEL> (pos = fma(scale, x, 0.5); floor;
                             Linear interpolation weights) + grid_index<N_DIMS,HASH_TYPE>() (stride walk while
                             stride <= hashmap_size, else coherent_prime_hash: primes 1, 2654435761, 805459861;
                             `% hashmap_size`)
  HashGridEncoding           grid.h kernel_grid output layout [level][feature] + bindings/torch/tinycudann/modules.py
                             Module.forward (input cast to float, params fp32 -> half per call, batch padded to 128)
  IdentityEncoding           include/tiny-cuda-nn/encodings/identity.h: identity() kernel, padded outputs = 1.0
  Network / fused_mlp        src/fully_fused_mlp.cu: kernel_mlp_fused / threadblock_layer (no bias, ReLU hidden, half
                             accumulators), include/tiny-cuda-nn/networks/fully_fused_mlp.h (weight matrices [out,in]
                             row-major, consecutive; padded_output_width = next_multiple(n_out, 16)),
                             src/network.cu / network_with_input_encoding.h (encoding alignment to 16)
  Network init               fully_fused_mlp.cu: initialize_params -> xavier_uniform per matrix; grid: U(-1e-4, 1e-4)
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List

import numpy as np
import torch
from torch import nn

PRIME_Y = 2654435761
PRIME_Z = 805459861
U32 = 0xFFFFFFFF


class Precision:
    """Where fp16 roundings are applied.

    mode "reference": every rounding tcnn applies (half interpolation fma, half output,
                      half MLP activations) -- closest to what the reference executes.
    mode "kernel":    the roundings of the CUDA kernels: fp16-stored tables and weights,
                      fp32 interpolation/blend, activations rounded to fp16 between
                      MLP layers, fp32 accumulation.
    mode "none":      fp16-stored tables/weights only; all math fp32.
    """
    mode = "reference"
    autocast = False   # emulate torch.autocast(fp16) around nn.Linear (training only in the reference)


@dataclass
class GridLevels:
    n_levels: int
    scale: np.ndarray      # float32 [L]
    res: np.ndarray        # int64 [L]
    entries: np.ndarray    # int64 [L]   (params_in_level / n_features)
    offset: np.ndarray     # int64 [L+1] (entry units)
    hashed: np.ndarray     # bool  [L]

    @property
    def total_entries(self) -> int:
        return int(self.offset[-1])


def hashgrid_levels(n_levels=16, log2_hashmap_size=19, base_resolution=16,
                    per_level_scale=1.4472692012786865) -> GridLevels:
    """grid.h: scale_l = exp2f(l*log2f(s))*base - 1 (float32); res = ceil(scale)+1;
    params_in_level = min(next_multiple(res^3, 8), 2^log2T); offsets = running sum."""
    s = np.float32(per_level_scale)
    l2 = np.log2(s)  # float32
    scale, res, ent, off, hashed = [], [], [], [0], []
    for l in range(n_levels):
        sc = np.float32(np.exp2(np.float32(l) * l2) * np.float32(base_resolution) - np.float32(1.0))
        r = int(np.ceil(sc)) + 1
        dense = ((r ** 3 + 7) // 8) * 8
        e = min(dense, 1 << log2_hashmap_size)
        # grid_index: hashed iff hashmap_size < stride after the stride walk
        stride = 1
        for _ in range(3):
            if stride <= e:
                stride *= r
        scale.append(sc); res.append(r); ent.append(e); off.append(off[-1] + e); hashed.append(e < stride)
    return GridLevels(n_levels, np.array(scale, np.float32), np.array(res, np.int64),
                      np.array(ent, np.int64), np.array(off, np.int64), np.array(hashed, bool))


def hashgrid_indices_weights(x: torch.Tensor, lv: GridLevels):
    """kernel_grid index/weight computation for Linear interpolation.

    x [B,3] float32 in [0,1).  Returns idx int64 [B,L,8] (entry index incl. level offset)
    and w float32 [B,L,8] (differentiable w.r.t. x).  Corner c has bit d set => +1 in dim d.
    pos = fmaf(scale, x, 0.5) (emulated in float64 then rounded), g = floor(pos), w = pos - g.
    """
    B = x.shape[0]
    idxs, ws = [], []
    for l in range(lv.n_levels):
        scale = float(lv.scale[l])
        res = int(lv.res[l]); ent = int(lv.entries[l]); off = int(lv.offset[l])
        with torch.no_grad():
            pos_ng = (x.detach().double() * scale + 0.5).float()
            g = torch.floor(pos_ng)
            gi = g.long()
        # fractional part: value from the fmaf emulation, gradient d frac / d x = scale
        frac = (pos_ng - g) + scale * (x - x.detach())
        lidx, lw = [], []
        for c in range(8):
            d = [(c >> k) & 1 for k in range(3)]
            cx = gi[:, 0] + d[0]; cy = gi[:, 1] + d[1]; cz = gi[:, 2] + d[2]
            wgt = None
            for k in range(3):
                a = frac[:, k] if d[k] else (1.0 - frac[:, k])
                wgt = a if wgt is None else wgt * a
            if lv.hashed[l]:
                index = (cx & U32) ^ ((cy * PRIME_Y) & U32) ^ ((cz * PRIME_Z) & U32)
            else:
                # stride walk (all three dims fit for dense levels)
                index = (cx + cy * res + cz * res * res) & U32
            index = index % ent
            lidx.append(index + off); lw.append(wgt)
        idxs.append(torch.stack(lidx, -1)); ws.append(torch.stack(lw, -1))
    return torch.stack(idxs, 1), torch.stack(ws, 1)


def half_round(t: torch.Tensor) -> torch.Tensor:
    """Round to fp16 and return as float32 (straight-through gradient)."""
    return t + (t.half().float() - t).detach()


class HashGridEncoding(nn.Module):
    """tcnn.Encoding(3, {"otype":"HashGrid", ...}).  params: flat fp32
    [(offset_l + idx) * F + f]; init U(-1e-4, 1e-4); forward casts params to fp16."""

    def __init__(self, n_input_dims: int, cfg: dict, seed: int = 1337):
        super().__init__()
        assert n_input_dims == 3
        assert cfg.get("interpolation", "Linear") == "Linear"
        self.F = int(cfg["n_features_per_level"])
        self.lv = hashgrid_levels(int(cfg["n_levels"]), int(cfg["log2_hashmap_size"]),
                                  int(cfg["base_resolution"]), float(cfg["per_level_scale"]))
        self.n_output_dims = self.lv.n_levels * self.F
        g = torch.Generator().manual_seed(seed)
        p = (torch.rand(self.lv.total_entries * self.F, generator=g) * 2 - 1) * 1e-4
        self.params = nn.Parameter(p)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x.float()
        idx, w = hashgrid_indices_weights(x, self.lv)          # [B,L,8]
        table = half_round(self.params).view(-1, self.F)        # fp16-stored
        B, L, _ = idx.shape
        vals = table[idx.reshape(-1)].view(B, L, 8, self.F)
        if Precision.mode == "reference":
            # result = fma((half)w, val, result) in half, corner order 0..7
            acc = torch.zeros(B, L, self.F)
            for c in range(8):
                acc = half_round(half_round(w[:, :, c, None]) * vals[:, :, c] + acc)
            out = acc
        else:
            out = (w[..., None] * vals).sum(2)
        out = out.reshape(B, L * self.F)
        if Precision.mode == "reference":
            return out.half()
        return out


class IdentityEncoding(nn.Module):
    def __init__(self, n_input_dims: int, cfg: dict):
        super().__init__()
        self.n_output_dims = n_input_dims
        self.params = nn.Parameter(torch.zeros(0))

    def forward(self, x):
        return x.half() if Precision.mode == "reference" else x.float()


class FrequencyEncoding(nn.Module):
    """Constructed by the reference field (nersemble_nerfacto_field.py:132-135) but never
    evaluated on this path (use_pred_normals=False)."""

    def __init__(self, n_input_dims: int, cfg: dict):
        super().__init__()
        self.n_output_dims = n_input_dims * 2 * int(cfg.get("n_frequencies", 12))
        self.params = nn.Parameter(torch.zeros(0))

    def forward(self, x):
        raise NotImplementedError("Frequency encoding is off the hot path")


def Encoding(n_input_dims: int, encoding_config: dict, seed: int = 1337, dtype=None):
    otype = encoding_config["otype"]
    if otype == "HashGrid":
        return HashGridEncoding(n_input_dims, encoding_config, seed)
    if otype == "Identity":
        return IdentityEncoding(n_input_dims, encoding_config)
    if otype == "Frequency":
        return FrequencyEncoding(n_input_dims, encoding_config)
    raise NotImplementedError(otype)


def _ceil_to(x, m):
    return ((x + m - 1) // m) * m


class Network(nn.Module):
    """tcnn.Network(n_in, n_out, {"otype":"FullyFusedMLP", ...}) = identity encoding that pads
    the input to a multiple of 16 with 1.0 + bias-free fp16 MLP; output padded to 16, sliced."""

    def __init__(self, n_input_dims: int, n_output_dims: int, network_config: dict, seed: int = 1337):
        super().__init__()
        assert network_config["otype"] == "FullyFusedMLP"
        assert network_config["activation"] == "ReLU"
        self.n_input_dims = n_input_dims
        self.n_output_dims = n_output_dims
        self.in_pad = _ceil_to(n_input_dims, 16)
        self.out_pad = _ceil_to(n_output_dims, 16)
        self.width = int(network_config["n_neurons"])
        self.n_hidden = int(network_config["n_hidden_layers"])
        self.out_act = network_config["output_activation"]
        self.shapes: List[tuple] = [(self.width, self.in_pad)]
        self.shapes += [(self.width, self.width)] * (self.n_hidden - 1)
        self.shapes += [(self.out_pad, self.width)]
        g = torch.Generator().manual_seed(seed)
        chunks = []
        for (o, i) in self.shapes:
            bound = math.sqrt(6.0 / (i + o))
            chunks.append(((torch.rand(o * i, generator=g) * 2 - 1) * bound))
        self.params = nn.Parameter(torch.cat(chunks))

    def weights(self) -> List[torch.Tensor]:
        out, ofs = [], 0
        for (o, i) in self.shapes:
            out.append(self.params[ofs:ofs + o * i].view(o, i)); ofs += o * i
        return out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        B = x.shape[0]
        x = x.float()
        if self.in_pad > self.n_input_dims:
            x = torch.cat([x, torch.ones(B, self.in_pad - self.n_input_dims)], -1)
        rnd = Precision.mode in ("reference", "kernel")
        h = half_round(x) if rnd else x
        ws = self.weights()
        for li, W in enumerate(ws):
            Wh = half_round(W)
            h = h @ Wh.t()
            last = li == len(ws) - 1
            if not last:
                h = torch.relu(h)
                if rnd:
                    h = half_round(h)
        if self.out_act == "Sigmoid":
            if Precision.mode == "reference":
                h = half_round(h)
            h = torch.sigmoid(h)
        elif self.out_act != "None":
            raise NotImplementedError(self.out_act)
        h = h[:, : self.n_output_dims]
        if Precision.mode == "reference":
            return h.half()
        return h


class NetworkWithInputEncoding(Network):
    def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, seed: int = 1337):
        assert encoding_config["otype"] == "Identity", "only Identity is used on this path"
        super().__init__(n_input_dims, n_output_dims, network_config, seed)
